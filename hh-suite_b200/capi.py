"""ctypes binding of the C-ABI in include/hhg.h (the only way Python reaches the kernels).

The classes mirror the reference's objects on this path:
  Context  ~ one ViterbiRunner worker (stream + scratch)        src/hhviterbirunner.h:52
  TargetDB ~ the HMMSimd batches of the whole shard, resident   src/hhhmmsimd.h:8
  Plan     ~ one ViterbiRunner::alignment call over a target list
There is no CPU fallback: loading fails loudly when the library or a GPU is missing.
"""
from __future__ import annotations

import ctypes as C
import os
import re

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
HEADER = os.path.join(os.path.dirname(HERE), "include", "hhg.h")

c_f32p = C.POINTER(C.c_float)
c_i32p = C.POINTER(C.c_int32)
c_i64p = C.POINTER(C.c_int64)
c_u8p = C.POINTER(C.c_uint8)
c_f64p = C.POINTER(C.c_double)


class Params(C.Structure):
    _fields_ = [("local", C.c_int), ("egq", C.c_float), ("egt", C.c_float), ("shift", C.c_float),
                ("ssw", C.c_float), ("use_ss", C.c_int), ("corr", C.c_float), ("ssm", C.c_int)]


HIT_DTYPE = np.dtype([("score", np.float32), ("i2", np.int32), ("j2", np.int32), ("i1", np.int32),
                      ("j1", np.int32), ("nsteps", np.int32), ("matched_cols", np.int32),
                      ("path_off", np.int32), ("hit_score", np.float32), ("score_ss", np.float32)])


class PrepParams(C.Structure):
    """hhg_prep_params: Parameters::gap* and pc_hhm_nocontext_* handed to PrepareTemplateHMM (src/hhfunc.cpp:170-178);
    defaults = src/hhdecl.cpp:64-80."""
    _fields_ = [("gapb", C.c_float), ("gapd", C.c_float), ("gape", C.c_float), ("gapf", C.c_float),
                ("gapg", C.c_float), ("gaph", C.c_float), ("gapi", C.c_float), ("pcm", C.c_int32),
                ("pca", C.c_float), ("pcb", C.c_float), ("pcc", C.c_float)]

    @classmethod
    def defaults(cls):
        return cls(1.0, 0.15, 1.0, 0.6, 0.6, 0.6, 0.6, 2, 1.0, 1.5, 1.0)


class MsaParams(C.Structure):
    """hhg_msa_params: the Parameters the A3M branch of HHEntry::getTemplateHMM reads (src/hhdatabase.cpp:441-449;
    defaults src/hhdecl.cpp:10-14,35-46,131-135).  M: 1 A2M/A3M (upper case = match), 2 gap percentage (Mgaps), 3 first
    sequence; wg: 0 position-specific weights, 1 global weights."""
    _fields_ = [("maxseq", C.c_int32), ("maxcol", C.c_int32), ("maxres", C.c_int32), ("M", C.c_int32), ("mark", C.c_int32),
                ("max_seqid", C.c_int32), ("coverage", C.c_int32), ("qid", C.c_int32), ("Ndiff", C.c_int32),
                ("qsc", C.c_float), ("wg", C.c_int32), ("Mgaps", C.c_int32)]

    @classmethod
    def defaults(cls, **kw):
        mp = cls()
        load().hhg_msa_params_default(C.byref(mp))
        for k, v in kw.items():
            setattr(mp, k, v)
        return mp


class Admix(C.Structure):
    """hhg_admix: pseudocount admixture tau(Neff) of cs::Admix (src/cs/pseudocounts.h:52-115).
    kind 0 constant, 1 CS-BLAST (prefilter default 0.8 / 2.0), 2 HHsearch (query HMM default 0.9 / 4.0 / 1.0)."""
    _fields_ = [("kind", C.c_int32), ("pca", C.c_double), ("pcb", C.c_double), ("pcc", C.c_double)]

    @classmethod
    def hhm(cls):
        return cls(2, 0.90, 4.00, 1.0)        # par.pc_hhm_context_engine, src/hhdecl.cpp:52-56

    @classmethod
    def prefilter(cls):
        return cls(1, 0.80, 2.00, 1.0)        # par.pc_prefilter_context_engine, :58-62


class Crf:
    """hhg_crf: the context library of the CRF pseudocounts (text of a `.crf` file, e.g. HH-suite's context_data.crf)."""

    def __init__(self, ctx, text: bytes):
        self._open(ctx, "hhg_crf_parse_host", "hhg_crf_create", text)

    def _open(self, ctx, parse_host, create, text, *args):
        """Host-only handle (ctx None) or one uploaded to ctx's device, then its size."""
        self.h = C.c_void_p()
        self.ctx = ctx
        if ctx is None:
            _ck(getattr(load(), parse_host)(text, len(text), *args, C.byref(self.h)))
        else:
            _ck(getattr(ctx.L, create)(ctx.h, text, len(text), *args, C.byref(self.h)))
        n = np.zeros(1, np.int32); w = np.zeros(1, np.int32)
        _ck(load().hhg_crf_info(self.h, _p(n, c_i32p), _p(w, c_i32p), None))
        self.n_states, self.window = int(n[0]), int(w[0])

    def pc(self):
        out = np.zeros((self.n_states, 20), np.float64)
        n = np.zeros(1, np.int32); w = np.zeros(1, np.int32)
        _ck(load().hhg_crf_info(self.h, _p(n, c_i32p), _p(w, c_i32p), _p(out, c_f64p)))
        return out

    def state(self, k):
        w = np.zeros((self.window, 20), np.float64); b = C.c_double()
        _ck(load().hhg_crf_state(self.h, k, _p(w, c_f64p), C.byref(b)))
        return w, b.value

    def tail_host(self, score, f, neff_m, admix):
        """Host only: the per-column log-sum-exp / admixture tail on given context scores [L, n_states]."""
        f = np.ascontiguousarray(f, np.float32); neff_m = np.ascontiguousarray(neff_m, np.float32)
        score = np.ascontiguousarray(score, np.float64).copy()
        L = f.shape[0] - 2
        p = np.zeros((L + 2, 20), np.float32)
        _ck(load().hhg_crf_tail_host(self.h, L, _p(score, c_f64p), _p(f, c_f32p), _p(neff_m, c_f32p), C.byref(admix), _p(p, c_f32p)))
        return p

    def pseudocounts(self, f, neff_m, neff_hmm, pb, admix, want_pav=True):
        """hhg_query_context_pseudocounts -> (p[(L+2),20] incl. rows 0 / L+1 = pav, pav[20]); without want_pav the
        background step is skipped: rows 0 and L+1 stay zero and pav is None."""
        f = np.ascontiguousarray(f, np.float32); neff_m = np.ascontiguousarray(neff_m, np.float32)
        pb = np.ascontiguousarray(pb, np.float32)
        L = f.shape[0] - 2
        p = np.zeros((L + 2, 20), np.float32); pav = np.zeros(20, np.float32) if want_pav else None
        _ck(self.ctx.L.hhg_query_context_pseudocounts(self.ctx.h, self.h, L, _p(f, c_f32p), _p(neff_m, c_f32p), float(neff_hmm),
                                                      _p(pb, c_f32p), C.byref(admix), _p(p, c_f32p), _p(pav, c_f32p)))
        return p, pav

    def close(self):
        if self.h:
            load().hhg_crf_destroy(self.h)
            self.h = None


class ContextLibrary(Crf):
    """hhg_crf of the generative engine: a context library (text of a `.lib` file, e.g. HH-suite's context_data.lib)
    with the window weights of -csw / -csb.  hhblits keeps those as floats, so the defaults are float32(1.6) and
    float32(0.85).  state(k) gives a profile's log-probabilities and log prior; pc() the central columns."""

    def __init__(self, ctx, text: bytes, weight_center=float(np.float32(1.6)), weight_decay=float(np.float32(0.85))):
        self.weight_center, self.weight_decay = float(weight_center), float(weight_decay)
        self._open(ctx, "hhg_context_library_parse_host", "hhg_context_library_create", text, self.weight_center,
                   self.weight_decay)


class SeqDb(C.Structure):
    """hhg_seqdb: `<db>_sequence.ffdata` + the offset / length columns of its `.ffindex` in index-file order."""
    _fields_ = [("n", C.c_int64), ("data", C.c_void_p), ("off", C.c_void_p), ("len", C.c_void_p)]

    @classmethod
    def make(cls, data: bytes, offsets, lengths):
        self = cls()
        self._buf = np.frombuffer(data, np.uint8)
        self._off = np.ascontiguousarray(offsets, np.int64); self._len = np.ascontiguousarray(lengths, np.int64)
        self.n = len(self._off); self.data = self._buf.ctypes.data; self.off = self._off.ctypes.data; self.len = self._len.ctypes.data
        return self


# one 112-byte column record of the resident database (include/hhg.h, hhg_db_read_cols)
COLREC_DTYPE = np.dtype([("p", np.float32, 20), ("m2m", np.float32), ("m2d", np.float32), ("d2m", np.float32),
                         ("d2d", np.float32), ("i2m", np.float32), ("i2i", np.float32), ("m2i", np.float32),
                         ("ss", np.uint32)])
assert COLREC_DTYPE.itemsize == 112


class MacParams(C.Structure):
    """hhg_mac_params: par.loc, par.shift, par.mact."""
    _fields_ = [("local", C.c_int32), ("shift", C.c_float), ("mact", C.c_float)]


# hhg_topk_rec: one record of the merged multi-GPU hit list (include/hhg.h)
TOPK_DTYPE = np.dtype([("target", np.int32), ("owner", np.int32), ("hit", HIT_DTYPE), ("key", np.uint64)])
assert TOPK_DTYPE.itemsize == 56

MAC_HIT_DTYPE = np.dtype([("i1", np.int32), ("i2", np.int32), ("j1", np.int32), ("j2", np.int32), ("nsteps", np.int32),
                          ("matched_cols", np.int32), ("sum_of_probs", np.float32), ("flags", np.int32),
                          ("pforward", np.float64), ("path_off", np.int64)])
assert MAC_HIT_DTYPE.itemsize == 48


class HhgError(RuntimeError):
    pass


def _p(a, t):
    return None if a is None else a.ctypes.data_as(t)


def _norm_type(decl: str) -> str:
    """A C type without const, one '*' per level of indirection: "const float* const*" -> "float**"."""
    words = [w for w in re.findall(r"\w+|\*", decl) if w != "const"]
    return " ".join(w for w in words if w != "*") + "*" * words.count("*")


def _prototypes():
    """(return type, name, [(parameter type, parameter name)]) of every hhg_* prototype in include/hhg.h."""
    with open(HEADER) as f:
        src = re.sub(r"/\*.*?\*/|//[^\n]*", " ", f.read(), flags=re.S)
    protos = []
    for ret, name, params in re.findall(r"([\w\s*]+?)\b(hhg_\w+)\s*\(([^()]*)\)\s*;", src):
        args = [] if params.strip() in ("", "void") else [re.fullmatch(r"\s*(.*?)\b(\w+)\s*", p).groups()
                                                            for p in params.split(",")]
        protos.append((_norm_type(ret), name, [(_norm_type(t), a) for t, a in args]))
    return protos


PROTOTYPES = _prototypes()
SYMBOLS = tuple(name for _, name, _ in PROTOTYPES)

# The ctypes type of each C type in include/hhg.h.  Beyond these tables, hhg_<handle>** (the out-parameter of every
# *_create) is POINTER(c_void_p) and any other pointer is c_void_p; any other type is refused.
_ARGTYPES = {"int": C.c_int, "int32_t": C.c_int, "int64_t": C.c_int64, "long long": C.c_longlong, "size_t": C.c_size_t,
             "float": C.c_float, "double": C.c_double, "float*": c_f32p, "int*": c_i32p, "int32_t*": c_i32p,
             "int64_t*": c_i64p, "uint8_t*": c_u8p, "double*": c_f64p, "char*": C.c_char_p,
             "hhg_params*": C.POINTER(Params), "hhg_prep_params*": C.POINTER(PrepParams),
             "hhg_mac_params*": C.POINTER(MacParams)}
_RESTYPES = {"int": C.c_int, "long long": C.c_longlong, "float": C.c_float, "double": C.c_double,
             "char*": C.c_char_p, "void": None}


def _ctypes_type(t: str, table: dict, what: str):
    if t in table:
        return table[t]
    if re.fullmatch(r"hhg_\w+\*\*", t):
        return C.POINTER(C.c_void_p)
    if t.endswith("*"):
        return C.c_void_p
    raise HhgError(f"include/hhg.h: {what} has type '{t}', which the binding does not map")


_lib = None


def lib_path() -> str:
    return os.path.join(HERE, "libhhg.so")


def load():
    """Load libhhg.so (building it first if a toolchain is present) and bind every prototype of include/hhg.h.
    Never falls back to CPU code."""
    global _lib
    if _lib is not None:
        return _lib
    from . import build as _build
    path = os.environ.get("HHG_LIB") or _build.build()   # HHG_LIB: developer override (kernel variants)
    L = C.CDLL(path)
    for ret, name, params in PROTOTYPES:
        fn = getattr(L, name)
        fn.restype = _ctypes_type(ret, _RESTYPES, f"the return value of {name}")
        fn.argtypes = [_ctypes_type(t, _ARGTYPES, f"parameter {a} of {name}") for t, a in params]
    _lib = L
    return L


def _ck(rc):
    if rc != 0:
        raise HhgError(f"hhg error {rc}: {load().hhg_last_error().decode()}")


class Context:
    def __init__(self, device: int = -1, stream: int | None = None):
        self.L = load()
        h = C.c_void_p()
        _ck(self.L.hhg_ctx_create(device, C.c_void_p(stream) if stream else None, C.byref(h)))
        self.h = h
        self.Lq = 0

    def close(self):
        if self.h:
            self.L.hhg_ctx_destroy(self.h)
            self.h = None

    def sync(self):
        _ck(self.L.hhg_ctx_sync(self.h))

    @property
    def launches(self) -> int:
        return int(self.L.hhg_ctx_launch_count(self.h))

    def fastlog2_table(self):
        out = np.zeros(1025, np.float32)
        _ck(self.L.hhg_debug_fastlog2_table(self.h, _p(out, c_f32p)))
        return out

    def set_excluded_regions(self, query_ranges=(), template_ranges=()):
        """-excl / -template_excl: lists of (lo, hi) 1-based inclusive ranges; empty lists clear."""
        q = np.array(query_ranges, np.int32).reshape(-1, 2); t = np.array(template_ranges, np.int32).reshape(-1, 2)
        ql, qh = np.ascontiguousarray(q[:, 0]), np.ascontiguousarray(q[:, 1])
        tl, th = np.ascontiguousarray(t[:, 0]), np.ascontiguousarray(t[:, 1])
        _ck(self.L.hhg_set_excluded_regions(self.h, len(q), _p(ql, c_i32p), _p(qh, c_i32p), len(t), _p(tl, c_i32p),
                                            _p(th, c_i32p)))

    def set_scwin(self, half_window: int):
        """-scwin: the half window D of column score 5 (the local amino-acid composition correction) for every following
        call of this context that applies it; default 40, D >= 1."""
        _ck(self.L.hhg_set_scwin(self.h, int(half_window)))

    def set_query(self, p, tr, ss=None, S33=None, local=True, egq=0.0, egt=0.0, shift=-0.03, ssw=0.11,
                  use_ss=False, corr=0.1, ssm=2):
        p = np.ascontiguousarray(p, np.float32); tr = np.ascontiguousarray(tr, np.float32)
        Lq = p.shape[0] - 2
        assert tr.shape[0] == Lq + 1
        ss = None if ss is None else np.ascontiguousarray(ss, np.uint8)
        S33 = None if S33 is None else np.ascontiguousarray(S33, np.float32)
        par = Params(1 if local else 0, egq, egt, shift, ssw, 1 if use_ss else 0, corr, ssm)
        _ck(self.L.hhg_query_set(self.h, Lq, _p(p, c_f32p), _p(tr, c_f32p), _p(ss, c_u8p), _p(S33, c_f32p),
                                 C.byref(par)))
        self.Lq = Lq


def query_local_background(ctx, p, pb):
    """Column score 5 for a query (PrepareQueryHMM under -sc 5): HMM::p [(L+2), 20] divided, rows 1..L, by the square
    root of its local background with the context's half window (Context.set_scwin) and the background pb[20].  Returns
    a new array; rows 0 and L+1 are copied unchanged."""
    out = np.array(p, np.float32, copy=True, order="C")
    pb = np.ascontiguousarray(pb, np.float32)
    assert out.ndim == 2 and out.shape[1] == 20 and pb.shape == (20,)
    _ck(ctx.L.hhg_query_local_background(ctx.h, out.shape[0] - 2, _p(pb, c_f32p), _p(out, c_f32p)))
    return out


def log2lin(tr):
    """HMM::Log2LinTransitionProbs(1.0) on a host array (through the C library's pow, like the reference)."""
    tr = np.ascontiguousarray(tr, np.float32)
    out = np.empty_like(tr)
    _ck(load().hhg_log2lin(tr.size, _p(tr, c_f32p), _p(out, c_f32p)))
    return out


def mac_query_set(ctx, q_p, q_tr_lin):
    """Query for MAC realignment: HMM::p and the LINEAR transitions (log2lin(q_tr))."""
    q_p = np.ascontiguousarray(q_p, np.float32); q_tr_lin = np.ascontiguousarray(q_tr_lin, np.float32)
    Lq = q_p.shape[0] - 2
    assert q_tr_lin.shape == (Lq + 1, 7)
    _ck(ctx.L.hhg_mac_query_set(ctx.h, Lq, _p(q_p, c_f32p), _p(q_tr_lin, c_f32p)))
    ctx.mac_Lq = Lq
    ctx.mac_batch_Lq = np.array([Lq], np.int32)


def mac_query_set_batch(ctx, queries, q_pav=None):
    """Queries for hhg_mac_realign_batch: queries = list of (HMM::p, LINEAR transitions); q_pav [nq, 20] (HMM::pav of
    each query) for realignments over a raw shard."""
    nq = len(queries)
    ps = [np.ascontiguousarray(q[0], np.float32) for q in queries]
    trs = [np.ascontiguousarray(q[1], np.float32) for q in queries]
    Lq = np.array([p.shape[0] - 2 for p in ps], np.int32)
    for L, t in zip(Lq, trs):
        assert t.shape == (L + 1, 7)
    pp = (C.c_void_p * nq)(*[p.ctypes.data for p in ps])
    tp = (C.c_void_p * nq)(*[t.ctypes.data for t in trs])
    qv = None if q_pav is None else np.ascontiguousarray(q_pav, np.float32)
    _ck(ctx.L.hhg_mac_query_set_batch(ctx.h, nq, _p(Lq, c_i32p), pp, tp, _p(qv, c_f32p)))
    ctx.mac_Lq = int(Lq[0])
    ctx.mac_batch_Lq = Lq


def _mac_inputs(vits, excl):
    """vit[n,5], vit_off, vit_i, vit_j and (excl_off, excl_i, excl_j) or Nones, as hhg_mac_realign(_batch) takes them."""
    n = len(vits)
    vit = np.zeros((n, 5), np.int32)
    voff = np.zeros(n + 1, np.int64)
    for r, v in enumerate(vits):
        vit[r] = v[:5]
        voff[r + 1] = voff[r] + v[4]
    vi = np.zeros(max(int(voff[-1]), 1), np.int32); vj = np.zeros_like(vi)
    for r, v in enumerate(vits):
        ns = v[4]
        vi[voff[r]:voff[r + 1]] = np.asarray(v[5])[1:ns + 1]
        vj[voff[r]:voff[r + 1]] = np.asarray(v[6])[1:ns + 1]
    eoff = ei = ej = None
    if excl is not None:
        eoff = np.zeros(n + 1, np.int64)
        for r, e in enumerate(excl):
            eoff[r + 1] = eoff[r] + (len(e[0]) if e is not None else 0)
        ei = np.zeros(max(int(eoff[-1]), 1), np.int32); ej = np.zeros_like(ei)
        for r, e in enumerate(excl):
            if e is not None and len(e[0]):
                ei[eoff[r]:eoff[r + 1]] = e[0]; ej[eoff[r]:eoff[r + 1]] = e[1]
    return vit, voff, vi, vj, eoff, ei, ej


def _mac_paths(hits, oi, oj, os_, op):
    """Per request: dict(i, j, states, P_posterior) with 1-based step arrays, sliced from the output buffers."""
    paths = []
    for r in range(len(hits)):
        o, ns = int(hits["path_off"][r]), int(hits["nsteps"][r])
        paths.append(dict(i=oi[o:o + ns + 1].copy(), j=oj[o:o + ns + 1].copy(), states=os_[o:o + ns + 1].copy(),
                          P_posterior=op[o:o + ns + 1].copy()))
    return paths


def mac_realign(ctx, db, targets, vits, excl=None, local=True, shift=-0.03, mact=0.35):
    """PosteriorDecoder::realign for a batch of hits.  vits[r] = (i1, i2, j1, j2, nsteps, i_steps, j_steps) with
    1-based step arrays (Hit.i / Hit.j); excl[r] = (alt_i, alt_j) of earlier MAC alignments of that template or None.
    Returns (hits[MAC_HIT_DTYPE], list of dict(i, j, states, P_posterior) with 1-based step arrays)."""
    n = len(targets)
    targets = np.ascontiguousarray(targets, np.int32)
    vit, voff, vi, vj, eoff, ei, ej = _mac_inputs(vits, excl)
    cap = int(np.sum(ctx.mac_Lq + db.Lh[np.clip(targets, 0, db.n - 1)].astype(np.int64) + 2))
    hits = np.zeros(n, MAC_HIT_DTYPE)
    oi = np.zeros(cap, np.int32); oj = np.zeros(cap, np.int32); os_ = np.zeros(cap, np.uint8); op = np.zeros(cap, np.float32)
    pp = MacParams(1 if local else 0, shift, mact)
    _ck(ctx.L.hhg_mac_realign(ctx.h, db.h, n, _p(targets, c_i32p), _p(vit, c_i32p), _p(voff, c_i64p), _p(vi, c_i32p),
                              _p(vj, c_i32p), _p(eoff, c_i64p), _p(ei, c_i32p), _p(ej, c_i32p), C.byref(pp),
                              hits.ctypes.data_as(C.c_void_p), _p(oi, c_i32p), _p(oj, c_i32p), _p(os_, c_u8p),
                              _p(op, c_f32p), cap))
    return hits, _mac_paths(hits, oi, oj, os_, op)


def mac_realign_batch(ctx, db, req_query, targets, vits, excl=None, columnscore=1, pb=None, local=True, shift=-0.03,
                      mact=0.35):
    """hhg_mac_realign_batch: request r realigns query req_query[r] of the last mac_query_set_batch against
    targets[r]; vits / excl and the result as in mac_realign.  columnscore / pb: the null model of a raw shard (5: the
    local composition correction with the context's half window, applied to a copy; the queries divided by
    query_local_background)."""
    n = len(targets)
    rq = np.ascontiguousarray(req_query, np.int32); targets = np.ascontiguousarray(targets, np.int32)
    vit, voff, vi, vj, eoff, ei, ej = _mac_inputs(vits, excl)
    qL = ctx.mac_batch_Lq
    cap = int(np.sum(qL[np.clip(rq, 0, len(qL) - 1)].astype(np.int64) +
                     db.Lh[np.clip(targets, 0, db.n - 1)].astype(np.int64) + 2))
    hits = np.zeros(n, MAC_HIT_DTYPE)
    oi = np.zeros(cap, np.int32); oj = np.zeros(cap, np.int32); os_ = np.zeros(cap, np.uint8); op = np.zeros(cap, np.float32)
    pp = MacParams(1 if local else 0, shift, mact)
    pbv = None if pb is None else np.ascontiguousarray(pb, np.float32)
    _ck(ctx.L.hhg_mac_realign_batch(ctx.h, db.h, n, _p(rq, c_i32p), _p(targets, c_i32p), _p(vit, c_i32p),
                                    _p(voff, c_i64p), _p(vi, c_i32p), _p(vj, c_i32p), _p(eoff, c_i64p), _p(ei, c_i32p),
                                    _p(ej, c_i32p), columnscore, _p(pbv, c_f32p), C.byref(pp),
                                    hits.ctypes.data_as(C.c_void_p), _p(oi, c_i32p), _p(oj, c_i32p), _p(os_, c_u8p),
                                    _p(op, c_f32p), cap))
    return hits, _mac_paths(hits, oi, oj, os_, op)


def mac_debug_posterior(ctx, request, Lt):
    out = np.zeros((ctx.mac_Lq + 1, Lt + 1), np.float32)
    _ck(ctx.L.hhg_mac_debug_posterior(ctx.h, request, _p(out, c_f32p)))
    return out


def _query_from(L: int, has_ss: bool, fn, *args):
    """Shared body of query_from_hhm / query_from_a3m: fn(*args, L_cap, L_out, p, tr, ss, pav, neff) fills the arrays."""
    p = np.zeros((L + 2, 20), np.float32); tr = np.zeros((L + 1, 7), np.float32)
    ss = np.zeros(L + 2, np.uint8); pav = np.zeros(20, np.float32)
    neff = np.zeros(1, np.float32); Lo = np.zeros(1, np.int32)
    _ck(fn(*args, L, _p(Lo, c_i32p), _p(p, c_f32p), _p(tr, c_f32p), _p(ss, c_u8p), _p(pav, c_f32p), _p(neff, c_f32p)))
    return dict(L=L, p=p, tr=tr, ss=ss, pav=pav, neff=float(neff[0]), has_ss=has_ss)


def query_from_hhm(ctx: "Context", record: bytes, R, params: "PrepParams | None" = None):
    """hhg_query_from_hhm: PrepareQueryHMM (nocontxt) of one HHM record -> dict(L, p, tr, ss, pav, neff)."""
    L, has_ss = hhm_scan(record)
    R = np.ascontiguousarray(R, np.float32)
    pp = params or PrepParams.defaults()
    return _query_from(L, has_ss, ctx.L.hhg_query_from_hhm, ctx.h, record, len(record), C.byref(pp), _p(R, c_f32p))


def a3m_scan(record: bytes, mp: "MsaParams | None" = None):
    """(match columns, sequences, has ss_pred) of one A3M record; host only."""
    mp = mp or MsaParams.defaults()
    L = np.zeros(1, np.int32); N = np.zeros(1, np.int32); ss = np.zeros(1, np.int32)
    _ck(load().hhg_a3m_scan(record, len(record), C.byref(mp), _p(L, c_i32p), _p(N, c_i32p), _p(ss, c_i32p)))
    return int(L[0]), int(N[0]), bool(ss[0])


def _msa_scan(record: bytes, seqs: "SeqDb | None", mp: "MsaParams"):
    """(match columns, sequences) of an A3M record, or of a compressed one when seqs is given; host only."""
    if seqs is None:
        return a3m_scan(record, mp)[:2]
    Lh = np.zeros(1, np.int32); Nh = np.zeros(1, np.int32)
    _ck(load().hhg_ca3m_scan(record, len(record), C.byref(seqs), C.byref(mp), _p(Lh, c_i32p), _p(Nh, c_i32p)))
    return int(Lh[0]), int(Nh[0])


def _msa_parse(record: bytes, seqs: "SeqDb | None", mp: "MsaParams | None"):
    """Shared body of a3m_parse / ca3m_parse (seqs given: compressed record)."""
    mp = mp or MsaParams.defaults()
    L, N = _msa_scan(record, seqs, mp)
    dims = np.zeros(6, np.int32)
    X = np.zeros((N, L + 2), np.uint8); I = np.zeros((N, L + 2), np.uint16); keep = np.zeros(N, np.int8)
    nres = np.zeros(N, np.int32); ksort = np.zeros(N, np.int32)
    out = (L, N, _p(dims, c_i32p), _p(X, c_u8p), I.ctypes.data, keep.ctypes.data, _p(nres, c_i32p), _p(ksort, c_i32p))
    if seqs is None:
        _ck(load().hhg_a3m_parse(record, len(record), C.byref(mp), *out))
    else:
        _ck(load().hhg_ca3m_parse(record, len(record), C.byref(seqs), C.byref(mp), *out))
    return dict(L=L, N_in=N, kfirst=int(dims[3]), kss_pred=int(dims[4]), kss_conf=int(dims[5]), X=X, I=I, keep=keep,
                nres=nres, ksort=ksort)


def a3m_parse(record: bytes, mp: "MsaParams | None" = None):
    """hhg_a3m_parse (host only): what Alignment::Read + Compress + the first steps of Filter2 hold for one record."""
    return _msa_parse(record, None, mp)


def ca3m_parse(record: bytes, seqs: "SeqDb", mp: "MsaParams | None" = None):
    """hhg_ca3m_parse (host only): a compressed-alignment record as Alignment::ReadCompressed + Compress hold it."""
    d = _msa_parse(record, seqs, mp)
    del d["kss_pred"], d["kss_conf"]
    return d


def _to_hmm(ctx: "Context", record: bytes, seqs: "SeqDb | None", pb, S, mp: "MsaParams | None"):
    """Shared body of msa_to_hmm / ca3m_to_hmm (seqs given: compressed record, whose ss row stays zero)."""
    mp = mp or MsaParams.defaults()
    L, N = _msa_scan(record, seqs, mp)
    dims = np.zeros(6, np.int32)
    keep = np.zeros(N, np.int8); wg = np.zeros(N, np.float32)
    f = np.zeros((L + 2, 20), np.float32); tr = np.zeros((L + 1, 7), np.float32); neff = np.zeros((3, L + 1), np.float32)
    nh = np.zeros(1, np.float32); ss = np.zeros(L + 2, np.uint8)
    pb = np.ascontiguousarray(pb, np.float32)
    Sm = None if S is None else np.ascontiguousarray(S, np.float32)
    out = (_p(Sm, c_f32p), _p(pb, c_f32p), L, N, _p(dims, c_i32p), keep.ctypes.data, _p(wg, c_f32p), _p(f, c_f32p),
           _p(tr, c_f32p), _p(neff, c_f32p), _p(nh, c_f32p))
    if seqs is None:
        _ck(ctx.L.hhg_msa_to_hmm(ctx.h, record, len(record), C.byref(mp), *out, _p(ss, c_u8p)))
    else:
        _ck(ctx.L.hhg_ca3m_to_hmm(ctx.h, record, len(record), C.byref(seqs), C.byref(mp), *out))
    return dict(L=L, N_in=N, N_filtered=int(dims[2]), kfirst=int(dims[3]), keep=keep, wg=wg, f=f, tr=tr, neff_m=neff[0],
                neff_i=neff[1], neff_d=neff[2], neff_hmm=float(nh[0]), ss=ss)


def ca3m_to_hmm(ctx: "Context", record: bytes, seqs: "SeqDb", pb, S=None, mp: "MsaParams | None" = None):
    """hhg_ca3m_to_hmm: one compressed-alignment record -> the raw HMM (see msa_to_hmm)."""
    return _to_hmm(ctx, record, seqs, pb, S, mp)


def msa_to_hmm(ctx: "Context", record: bytes, pb, S=None, mp: "MsaParams | None" = None):
    """hhg_msa_to_hmm: one A3M record -> the HMM Alignment::FrequenciesAndTransitions computes (no pseudocounts)."""
    return _to_hmm(ctx, record, None, pb, S, mp)


def query_from_a3m(ctx: "Context", record: bytes, R, pb, S=None, params: "PrepParams | None" = None,
                   mp: "MsaParams | None" = None):
    """hhg_query_from_a3m: query alignment -> HMM -> PrepareQueryHMM (nocontxt) -> dict(L, p, tr, ss, pav, neff)."""
    mp = mp or MsaParams.defaults()
    L, _, has_ss = a3m_scan(record, mp)
    R = np.ascontiguousarray(R, np.float32); pb = np.ascontiguousarray(pb, np.float32)
    Sm = None if S is None else np.ascontiguousarray(S, np.float32)
    pp = params or PrepParams.defaults()
    return _query_from(L, has_ss, ctx.L.hhg_query_from_a3m, ctx.h, record, len(record), C.byref(mp), _p(Sm, c_f32p),
                       _p(pb, c_f32p), C.byref(pp), _p(R, c_f32p))


def cs219_parse(text: bytes, n_cap: int = 256):
    """hhg_cs219_parse: the column-state library text (cs219.lib) -> float[n_states, 20] linear probabilities."""
    lib = np.zeros((n_cap, 20), np.float32)
    n = np.zeros(1, np.int32)
    _ck(load().hhg_cs219_parse(text, len(text), _p(lib, c_f32p), n_cap, _p(n, c_i32p)))
    return lib[:int(n[0])].copy()


def hhm_scan(record: bytes):
    """(LENG, has_ss_pred) of one HHM record; host only."""
    L = np.zeros(1, np.int32); ss = np.zeros(1, np.int32)
    _ck(load().hhg_hhm_scan(record, len(record), _p(L, c_i32p), _p(ss, c_i32p)))
    return int(L[0]), bool(ss[0])


def hhm_parse(record: bytes):
    """The integers of one HHM record as hhg_db_create_hhm tokenises them; host only."""
    L, has_ss = hhm_scan(record)
    f = np.zeros((L, 20), np.int32); trn = np.zeros((L + 1, 10), np.int32); ss = np.zeros(L, np.uint8)
    null = np.zeros(20, np.int32); neff = np.zeros(1, np.float32); has_pc = np.zeros(1, np.int32)
    _ck(load().hhg_hhm_parse(record, len(record), L, _p(f, c_i32p), _p(trn, c_i32p), _p(ss, c_u8p), _p(null, c_i32p),
                             _p(neff, c_f32p), _p(has_pc, c_i32p)))
    return dict(L=L, has_ss=has_ss, f=f, tr=trn[:, :7].copy(), neff=trn[:, 7:].copy(), ss=ss, null=null,
                neff_hmm=float(neff[0]), has_pc=int(has_pc[0]))


class TargetDB:
    """Device-resident shard of prepared target profiles (see synth.prepared_db for the host layout)."""

    def __init__(self, ctx: Context, L, p, tr, p_off, tr_off, ss=None, pav=None):
        """pav given: p holds pre-null-model emissions; call apply_null_model(q_pav) per query."""
        self.ctx = ctx
        self.Lh = np.ascontiguousarray(L, np.int32)
        n = len(self.Lh)
        p = np.ascontiguousarray(p, np.float32); tr = np.ascontiguousarray(tr, np.float32)
        po = np.ascontiguousarray(np.asarray(p_off, np.int64) * 20)
        to = np.ascontiguousarray(np.asarray(tr_off, np.int64) * 7)
        so = np.ascontiguousarray(np.asarray(p_off, np.int64))
        ss = None if ss is None else np.ascontiguousarray(ss, np.uint8)
        h = C.c_void_p()
        if pav is None:
            _ck(ctx.L.hhg_db_create(ctx.h, n, _p(self.Lh, c_i32p), _p(po, c_i64p), _p(to, c_i64p), _p(so, c_i64p),
                                    _p(p, c_f32p), _p(tr, c_f32p), _p(ss, c_u8p), C.byref(h)))
        else:
            pav = np.ascontiguousarray(pav, np.float32)
            assert pav.shape == (n, 20)
            _ck(ctx.L.hhg_db_create_raw(ctx.h, n, _p(self.Lh, c_i32p), _p(po, c_i64p), _p(to, c_i64p),
                                        _p(so, c_i64p), _p(p, c_f32p), _p(tr, c_f32p), _p(ss, c_u8p),
                                        _p(pav, c_f32p), C.byref(h)))
        self.h = h
        self.n = n

    @classmethod
    def _wrap(cls, ctx, h, n):
        self = cls.__new__(cls)
        self.ctx, self.h, self.n = ctx, h, n
        return self

    @classmethod
    def from_hhm(cls, ctx, data: bytes, offsets, lengths, R, params: "PrepParams | None" = None):
        """Build the shard from HHM text records (`_hhm.ffdata` bytes + the offset/length columns of its
        `.ffindex`): getTemplateHMM + the query-independent part of PrepareTemplateHMM, once per database.
        R: the 20x20 pseudocount matrix (R[a][b], SetSubstitutionMatrix).  Call apply_null_model per query."""
        R = np.ascontiguousarray(R, np.float32)
        assert R.shape == (20, 20)
        pp = params or PrepParams.defaults()
        return cls._from_records(ctx, data, offsets, lengths, ctx.L.hhg_db_create_hhm, C.byref(pp), _p(R, c_f32p))

    @classmethod
    def from_a3m(cls, ctx, data: bytes, offsets, lengths, R, pb, S=None, params: "PrepParams | None" = None,
                 mp: "MsaParams | None" = None):
        """Build the shard from A3M alignments (`_a3m.ffdata` bytes + offset/length columns): the alignment branch of
        getTemplateHMM (Read, Compress, Filter, FrequenciesAndTransitions) + the query-independent part of
        PrepareTemplateHMM, once per database.  pb: background frequencies, S: substitution matrix in bits (qsc only)."""
        return cls._from_msa(ctx, data, offsets, lengths, None, R, pb, S, params, mp)

    @classmethod
    def from_ca3m(cls, ctx, data: bytes, offsets, lengths, seqs: "SeqDb", R, pb, S=None, params: "PrepParams | None" = None,
                  mp: "MsaParams | None" = None):
        """Build the shard from a compressed alignment database (`_ca3m.ffdata` + `_sequence.ffdata`, see SeqDb)."""
        return cls._from_msa(ctx, data, offsets, lengths, seqs, R, pb, S, params, mp)

    @classmethod
    def _from_msa(cls, ctx, data: bytes, offsets, lengths, seqs, R, pb, S, params, mp):
        """Shared body of from_a3m / from_ca3m (seqs given: compressed records)."""
        R = np.ascontiguousarray(R, np.float32); pb = np.ascontiguousarray(pb, np.float32)
        Sm = None if S is None else np.ascontiguousarray(S, np.float32)
        pp = params or PrepParams.defaults()
        mp = mp or MsaParams.defaults()
        args = (C.byref(mp), _p(Sm, c_f32p), _p(pb, c_f32p), C.byref(pp), _p(R, c_f32p))
        if seqs is None:
            return cls._from_records(ctx, data, offsets, lengths, ctx.L.hhg_db_create_a3m, *args)
        return cls._from_records(ctx, data, offsets, lengths, ctx.L.hhg_db_create_ca3m, C.byref(seqs), *args)

    @classmethod
    def _from_records(cls, ctx, data: bytes, offsets, lengths, create, *args):
        """Shared body of the text-record loaders: create(ctx, n, data, offsets, lengths, *args, out) builds the shard."""
        off = np.ascontiguousarray(offsets, np.int64); ln = np.ascontiguousarray(lengths, np.int64)
        n = len(off)
        if n == 0 or len(ln) != n or off.min() < 0 or int((off + ln).max()) > len(data):
            raise ValueError("offsets/lengths do not fit the data buffer")
        h = C.c_void_p()
        buf = np.frombuffer(data, np.uint8)        # bytes or a (read-only) mmap of the ffdata file
        _ck(create(ctx.h, n, buf.ctypes.data_as(C.c_char_p), _p(off, c_i64p), _p(ln, c_i64p), *args, C.byref(h)))
        self = cls._wrap(ctx, h, n)
        self.Lh = np.zeros(n, np.int32)
        _ck(ctx.L.hhg_db_lengths(h, _p(self.Lh, c_i32p)))
        return self

    @classmethod
    def from_packed(cls, ctx, L, cols_raw, pav, has_ss=False):
        """Load the resident binary format written by read_cols(0) / read_pav()."""
        L = np.ascontiguousarray(L, np.int32)
        cols_raw = np.ascontiguousarray(cols_raw)
        assert cols_raw.dtype == COLREC_DTYPE and len(cols_raw) == int(L.sum())
        pav = np.ascontiguousarray(pav, np.float32)
        assert pav.shape == (len(L), 20)
        h = C.c_void_p()
        _ck(ctx.L.hhg_db_create_packed(ctx.h, len(L), _p(L, c_i32p), cols_raw.ctypes.data_as(C.c_void_p),
                                       1 if has_ss else 0, _p(pav, c_f32p), C.byref(h)))
        self = cls._wrap(ctx, h, len(L))
        self.Lh = L
        return self

    def read_cols(self, which=0, first=0, count=None):
        """Column records (COLREC_DTYPE): which=0 before the null model, 1 after apply_null_model."""
        total = int(self.ctx.L.hhg_db_columns(self.h))
        count = total - first if count is None else count
        out = np.zeros(count, COLREC_DTYPE)
        _ck(self.ctx.L.hhg_db_read_cols(self.ctx.h, self.h, which, first, count, out.ctypes.data_as(C.c_void_p)))
        return out

    def read_pav(self):
        out = np.zeros((self.n, 20), np.float32)
        _ck(self.ctx.L.hhg_db_read_pav(self.ctx.h, self.h, _p(out, c_f32p)))
        return out

    def apply_null_model(self, q_pav=None, pb=None, columnscore=1):
        """HMM::IncludeNullModelInHMM on the raw records: columnscore 0 pb, 1 (q_pav + t.pav)/2, 2 t.pav, 3 q_pav,
        5 the local composition correction (pb and the context's half window; q_pav is not used)."""
        q_pav = None if q_pav is None else np.ascontiguousarray(q_pav, np.float32)
        pb = None if pb is None else np.ascontiguousarray(pb, np.float32)
        _ck(self.ctx.L.hhg_db_apply_null_model(self.ctx.h, self.h, _p(q_pav, c_f32p), _p(pb, c_f32p), columnscore))

    @classmethod
    def from_profiles(cls, ctx, profiles):
        """profiles: list of (p[(L+2),20], tr[(L+1),7], ss[L+2]|None)."""
        L = np.array([q[0].shape[0] - 2 for q in profiles], np.int32)
        p_off = np.concatenate([[0], np.cumsum(L.astype(np.int64) + 2)[:-1]])
        tr_off = np.concatenate([[0], np.cumsum(L.astype(np.int64) + 1)[:-1]])
        P = np.concatenate([q[0] for q in profiles]).astype(np.float32)
        T = np.concatenate([q[1] for q in profiles]).astype(np.float32)
        has_ss = all(q[2] is not None for q in profiles)
        S = np.concatenate([q[2] for q in profiles]).astype(np.uint8) if has_ss else None
        return cls(ctx, L, P, T, p_off, tr_off, S)

    def close(self):
        if self.h:
            self.ctx.L.hhg_db_destroy(self.h)
            self.h = None


class HostStore:
    """The raw records of a whole database in page-locked, device-mapped host memory (hhg_dbstore): what a StagedDB
    stages from.  Targets are numbered in append order (global ids)."""

    def __init__(self, ctx: Context, capacity_targets: int, capacity_cols: int, has_ss: bool = False):
        self.ctx = ctx
        h = C.c_void_p()
        _ck(ctx.L.hhg_dbstore_create(ctx.h, capacity_targets, capacity_cols, 1 if has_ss else 0, C.byref(h)))
        self.h = h

    @property
    def n(self) -> int:
        return int(self.ctx.L.hhg_dbstore_size(self.h))

    @property
    def columns(self) -> int:
        return int(self.ctx.L.hhg_dbstore_columns(self.h))

    @property
    def Lh(self):
        out = np.zeros(self.n, np.int32)
        _ck(self.ctx.L.hhg_dbstore_lengths(self.h, _p(out, c_i32p)))
        return out

    def append_packed(self, L, cols_raw, pav):
        """Host arrays in the format TargetDB.read_cols(0) / read_pav() return."""
        L = np.ascontiguousarray(L, np.int32)
        cols_raw = np.ascontiguousarray(cols_raw)
        assert cols_raw.dtype == COLREC_DTYPE and len(cols_raw) == int(L.sum())
        pav = np.ascontiguousarray(pav, np.float32)
        assert pav.shape == (len(L), 20)
        _ck(self.ctx.L.hhg_dbstore_append_packed(self.h, len(L), _p(L, c_i32p), cols_raw.ctypes.data_as(C.c_void_p),
                                                 _p(pav, c_f32p)))

    def append_db(self, db: "TargetDB"):
        """All targets of a raw device shard (any loader): load a chunk, append it, close it."""
        _ck(self.ctx.L.hhg_dbstore_append_db(self.ctx.h, self.h, db.h))

    @classmethod
    def from_db(cls, ctx: Context, db: "TargetDB", has_ss: bool = False):
        self = cls(ctx, db.n, int(ctx.L.hhg_db_columns(db.h)), has_ss)
        self.append_db(db)
        return self

    def close(self):
        if self.h:
            _ck(self.ctx.L.hhg_dbstore_destroy(self.h))
            self.h = None


class RecordSource:
    """A database's own ffindex records (HHM, A3M or compressed A3M) as what a StagedDB stages from (hhg_recsrc): no
    record is parsed until a stage() call names it.  Global ids are record indices.  The data buffer (bytes or an mmap
    of the ffdata) and the SeqDb are kept referenced here and must stay valid while the source lives."""

    def __init__(self, ctx: Context, data: bytes, offsets, lengths, create, *args):
        """Shared body of the from_* constructors: create(ctx, n, data, offsets, lengths, *args, out)."""
        off = np.ascontiguousarray(offsets, np.int64); ln = np.ascontiguousarray(lengths, np.int64)
        n = len(off)
        if n == 0 or len(ln) != n or off.min() < 0 or ln.min() < 0 or int((off + ln).max()) > len(data):
            raise ValueError("offsets/lengths do not fit the data buffer")
        self.ctx, self._buf, self._off, self._len = ctx, np.frombuffer(data, np.uint8), off, ln
        h = C.c_void_p()
        _ck(create(ctx.h, n, self._buf.ctypes.data_as(C.c_char_p), _p(off, c_i64p), _p(ln, c_i64p), *args, C.byref(h)))
        self.h = h

    @classmethod
    def from_hhm(cls, ctx, data: bytes, offsets, lengths, R, params: "PrepParams | None" = None, has_ss: bool = False):
        """HHM records, with the arguments of TargetDB.from_hhm."""
        R = np.ascontiguousarray(R, np.float32)
        assert R.shape == (20, 20)
        pp = params or PrepParams.defaults()
        self = cls(ctx, data, offsets, lengths, ctx.L.hhg_recsrc_create_hhm, C.byref(pp), _p(R, c_f32p), 1 if has_ss else 0)
        self._keep = (pp, R)
        return self

    @classmethod
    def from_a3m(cls, ctx, data: bytes, offsets, lengths, R, pb, S=None, params: "PrepParams | None" = None,
                 mp: "MsaParams | None" = None, has_ss: bool = False):
        """A3M alignments, with the arguments of TargetDB.from_a3m."""
        return cls._from_msa(ctx, data, offsets, lengths, None, R, pb, S, params, mp, has_ss)

    @classmethod
    def from_ca3m(cls, ctx, data: bytes, offsets, lengths, seqs: "SeqDb", R, pb, S=None,
                  params: "PrepParams | None" = None, mp: "MsaParams | None" = None, has_ss: bool = False):
        """Compressed alignments, with the arguments of TargetDB.from_ca3m."""
        return cls._from_msa(ctx, data, offsets, lengths, seqs, R, pb, S, params, mp, has_ss)

    @classmethod
    def _from_msa(cls, ctx, data, offsets, lengths, seqs, R, pb, S, params, mp, has_ss):
        R = np.ascontiguousarray(R, np.float32); pb = np.ascontiguousarray(pb, np.float32)
        Sm = None if S is None else np.ascontiguousarray(S, np.float32)
        pp = params or PrepParams.defaults()
        mp = mp or MsaParams.defaults()
        args = (C.byref(mp), _p(Sm, c_f32p), _p(pb, c_f32p), C.byref(pp), _p(R, c_f32p), 1 if has_ss else 0)
        if seqs is None:
            self = cls(ctx, data, offsets, lengths, ctx.L.hhg_recsrc_create_a3m, *args)
        else:
            self = cls(ctx, data, offsets, lengths, ctx.L.hhg_recsrc_create_ca3m, C.byref(seqs), *args)
        self._keep = (seqs,)
        return self

    @property
    def n(self) -> int:
        return int(self.ctx.L.hhg_recsrc_size(self.h))

    def close(self):
        if self.h:
            _ck(self.ctx.L.hhg_recsrc_destroy(self.h))
            self.h = None


STAGE_STATS_DTYPE = np.dtype([("hits", np.int64), ("copied", np.int64), ("bytes", np.int64), ("evicted", np.int64)])


class StagedDB(TargetDB):
    """A TargetDB of max_targets slots that caches targets of a HostStore (hhg_db_create_staged) or builds them from a
    RecordSource's records when they are staged (hhg_db_create_staged_records); `store` is the one it was made over.
    Every TargetDB use works on it with LOCAL ids (slots); stage() makes targets resident, to_global() translates back.
    n is the number of slots, Lh the length of the target in each slot (0: empty)."""

    def __init__(self, ctx: Context, store: "HostStore | RecordSource", max_targets: int, max_cols: int):
        h = C.c_void_p()
        create = ctx.L.hhg_db_create_staged_records if isinstance(store, RecordSource) else ctx.L.hhg_db_create_staged
        _ck(create(ctx.h, store.h, max_targets, max_cols, C.byref(h)))
        self.ctx, self.h, self.n, self.store = ctx, h, max_targets, store
        self.Lh = np.zeros(max_targets, np.int32)
        self.last_stats = np.zeros(1, STAGE_STATS_DTYPE)[0]

    def stage(self, ids) -> np.ndarray:
        """Make the store's targets ids resident (hhg_db_stage); returns their local ids.  last_stats: what it cost."""
        ids = np.ascontiguousarray(ids, np.int32)
        local = np.zeros(len(ids), np.int32)
        stats = np.zeros(1, STAGE_STATS_DTYPE)
        _ck(self.ctx.L.hhg_db_stage(self.ctx.h, self.h, len(ids), _p(ids, c_i32p), _p(local, c_i32p),
                                    stats.ctypes.data_as(C.c_void_p)))
        self.last_stats = stats[0]
        _ck(self.ctx.L.hhg_db_lengths(self.h, _p(self.Lh, c_i32p)))
        return local

    def lookup(self, local):
        """(global ids, first arena column) of local ids; global id -1 = empty slot."""
        local = np.ascontiguousarray(local, np.int32)
        g = np.zeros(len(local), np.int32); first = np.zeros(len(local), np.int64)
        _ck(self.ctx.L.hhg_db_staged_lookup(self.h, len(local), _p(local, c_i32p), _p(g, c_i32p), _p(first, c_i64p)))
        return g, first

    def to_global(self, local) -> np.ndarray:
        return self.lookup(local)[0]

    def read_target(self, local: int):
        """Raw column records of the target in slot `local`."""
        return self.read_cols(0, int(self.lookup([local])[1][0]), int(self.Lh[local]))

    def neff(self, local) -> np.ndarray:
        """Neff_HMM of the targets in slots `local` (record-sourced shards only): the t_neff of hitlist_pvalues."""
        local = np.ascontiguousarray(local, np.int32)
        out = np.zeros(len(local), np.float32)
        _ck(self.ctx.L.hhg_db_staged_neff(self.h, len(local), _p(local, c_i32p), _p(out, c_f32p)))
        return out


class Comm:
    """hhg_comm: one rank of the NCCL communicator behind the C-ABI (world == 1: no NCCL involved)."""

    def __init__(self, ctx: Context, rank: int = 0, world: int = 1, unique_id: bytes | None = None):
        self.ctx, self.rank, self.world = ctx, rank, world
        h = C.c_void_p()
        buf = C.create_string_buffer(unique_id, 128) if unique_id is not None else None
        _ck(ctx.L.hhg_comm_create(ctx.h, rank, world, buf, C.byref(h)))
        self.h = h

    @staticmethod
    def unique_id() -> bytes:
        buf = C.create_string_buffer(128)
        _ck(load().hhg_comm_unique_id(buf))
        return buf.raw

    def close(self):
        if self.h:
            self.ctx.L.hhg_comm_destroy(self.h)
            self.h = None


def plan_topk(ctx: Context, plan_handle, comm: Comm | None, K: int, by_hit_score: bool = False, id_base: int = 0,
              global_ids=None):
    """hhg_plan_topk on a raw plan handle: the merged K best hit records (TOPK_DTYPE) on every rank."""
    out = np.zeros(K, TOPK_DTYPE)
    n = C.c_int32(0)
    gi = None if global_ids is None else np.ascontiguousarray(global_ids, np.int32)
    _ck(ctx.L.hhg_plan_topk(ctx.h, plan_handle, comm.h if comm is not None else None, K, 1 if by_hit_score else 0,
                            id_base, _p(gi, c_i32p), out.ctypes.data_as(C.c_void_p), C.byref(n)))
    return out[:n.value]


STATS_DTYPE = np.dtype([("Pval", np.float64), ("logPval", np.float64), ("Eval", np.float64), ("logEval", np.float64),
                        ("score_aass", np.float32), ("Probab", np.float32), ("lamda", np.float32), ("mu", np.float32)])


def hitlist_pvalues(score, score_ss, Lt, t_neff, Lq, q_neff, N_searched, loc=True, ssm=2, ssw=0.11, hit_has_ss=None):
    """HitList::CalculatePvalues on arrays (host side of the library): returns STATS_DTYPE records."""
    n = len(score)
    out = np.zeros(n, STATS_DTYPE)
    s = np.ascontiguousarray(score, np.float32); ss = np.ascontiguousarray(score_ss, np.float32)
    L = np.ascontiguousarray(Lt, np.int32); ne = np.ascontiguousarray(t_neff, np.float32)
    hs = None if hit_has_ss is None else np.ascontiguousarray(hit_has_ss, np.int32)
    _ck(load().hhg_hitlist_pvalues(n, _p(s, c_f32p), _p(ss, c_f32p), _p(L, c_i32p), _p(ne, c_f32p), _p(hs, c_i32p), Lq,
                                   q_neff, N_searched, 1 if loc else 0, ssm, ssw, out.ctypes.data_as(C.c_void_p)))
    return out


def hitlist_hhblits_evalues(stats, t_neff, q_neff, dbsize, alphaa=0.4, alphab=0.02, alphac=0.1, prefilter_evalue_thresh=1000.0):
    """HitList::CalculateHHblitsEvalues: overwrites Eval / logEval of `stats` in place."""
    ne = np.ascontiguousarray(t_neff, np.float32)
    _ck(load().hhg_hitlist_hhblits_evalues(len(stats), stats.ctypes.data_as(C.c_void_p), _p(ne, c_f32p), q_neff, dbsize,
                                           alphaa, alphab, alphac, prefilter_evalue_thresh))
    return stats


def early_stop_sum(score, Lt, t_neff, Lq, q_neff, prefilter=True, dbsize=1, alphaa=0.4, alphab=0.02, alphac=0.1,
                   prefilter_evalue_thresh=1000.0):
    """ViterbiRunner::calculateEarlyStop over one chunk of hits."""
    s = np.ascontiguousarray(score, np.float32); L = np.ascontiguousarray(Lt, np.int32)
    ne = np.ascontiguousarray(t_neff, np.float32)
    return float(load().hhg_early_stop_sum(len(s), _p(s, c_f32p), _p(L, c_i32p), _p(ne, c_f32p), Lq, q_neff,
                                           1 if prefilter else 0, dbsize, alphaa, alphab, alphac, prefilter_evalue_thresh))


def hitlist_order(stats, files=None):
    """HitList::SortList order (score_aass ascending, then file name)."""
    n = len(stats)
    order = np.zeros(n, np.int32)
    farr = None if files is None else (C.c_char_p * n)(*[f.encode() for f in files])
    _ck(load().hhg_hitlist_order(n, stats.ctypes.data_as(C.c_void_p), farr, _p(order, c_i32p)))
    return order


def plan_topk_by_key(ctx: Context, plan_handle, comm, K: int, key, id_base: int = 0, global_ids=None):
    """hhg_plan_topk_by_key: merged K best by a caller-supplied per-request value (ascending = better)."""
    out = np.zeros(K, TOPK_DTYPE)
    n = C.c_int32(0)
    key = np.ascontiguousarray(key, np.float32)
    gi = None if global_ids is None else np.ascontiguousarray(global_ids, np.int32)
    _ck(ctx.L.hhg_plan_topk_by_key(ctx.h, plan_handle, comm.h if comm is not None else None, K, _p(key, c_f32p), id_base,
                                   _p(gi, c_i32p), out.ctypes.data_as(C.c_void_p), C.byref(n)))
    return out[:n.value]


def plan_topk_paths(ctx: Context, plan_handle, comm: Comm | None, recs: np.ndarray, width: int | None = None):
    """hhg_plan_topk_paths: [len(recs), width] uint8 state strings of the merged list, zero padded."""
    recs = np.ascontiguousarray(recs)
    width = int(width or max(1, int(recs["hit"]["nsteps"].max()) if len(recs) else 1))
    out = np.zeros((len(recs), width), np.uint8)
    _ck(ctx.L.hhg_plan_topk_paths(ctx.h, plan_handle, comm.h if comm is not None else None, len(recs),
                                  recs.ctypes.data_as(C.c_void_p), width, _p(out, c_u8p)))
    return out


class Plan:
    def __init__(self, ctx: Context, db: TargetDB, ids=None):
        self.ctx, self.db = ctx, db
        self.ids = np.arange(db.n, dtype=np.int32) if ids is None else np.ascontiguousarray(ids, np.int32)
        self.n = len(self.ids)
        h = C.c_void_p()
        _ck(ctx.L.hhg_plan_create(ctx.h, db.h, self.n, _p(self.ids, c_i32p), C.byref(h)))
        self.h = h
        self.cells = ctx.L.hhg_plan_cells(h)
        self.padded_cells = ctx.L.hhg_plan_padded_cells(h)
        self.alg_bytes = ctx.L.hhg_plan_algorithmic_bytes(h)
        self.path_cap = int(np.sum(self.ctx.Lq + db.Lh[self.ids].astype(np.int64) + 2))

    def run(self):
        _ck(self.ctx.L.hhg_plan_run(self.ctx.h, self.h))

    def run_timed(self):
        """Returns (ms_viterbi_kernels, ms_backtrace_kernels) measured with CUDA events on the stream."""
        a = C.c_float(); b = C.c_float()
        _ck(self.ctx.L.hhg_plan_run_timed(self.ctx.h, self.h, C.byref(a), C.byref(b)))
        return a.value, b.value

    def fetch(self, want_paths=True, hits=None, paths=None):
        hits = np.zeros(self.n, HIT_DTYPE) if hits is None else hits
        if want_paths and paths is None:
            paths = np.zeros(self.path_cap, np.uint8)
        _ck(self.ctx.L.hhg_plan_fetch(self.ctx.h, self.h, hits.ctypes.data_as(C.c_void_p), _p(paths, c_u8p),
                                      self.path_cap if want_paths else 0))
        return hits, paths

    def topk(self, K, comm=None, by_hit_score=False, id_base=0, global_ids=None):
        return plan_topk(self.ctx, self.h, comm, K, by_hit_score, id_base, global_ids)

    def topk_paths(self, recs, comm=None, width=None):
        return plan_topk_paths(self.ctx, self.h, comm, recs, width)

    def debug_bt(self, k):
        Lt = int(self.db.Lh[self.ids[k]])
        bt = np.zeros((self.ctx.Lq + 1, Lt + 1), np.uint8)
        _ck(self.ctx.L.hhg_plan_debug_bt(self.ctx.h, self.h, k, _p(bt, c_u8p)))
        return bt

    def close(self):
        if self.h:
            self.ctx.L.hhg_plan_destroy(self.h)
            self.h = None


def _exclusions(exclusions):
    """(excl_off, excl_i, excl_j) of a per-request list of (i_steps, j_steps) or None entries; Nones without a list."""
    if exclusions is None:
        return None, None, None
    cnt = np.array([0 if e is None else len(e[0]) for e in exclusions], np.int64)
    eo = np.concatenate([[0], np.cumsum(cnt)]).astype(np.int64)
    ei = np.concatenate([np.asarray(e[0], np.int32) for e in exclusions if e is not None] or
                        [np.zeros(0, np.int32)]).astype(np.int32)
    ej = np.concatenate([np.asarray(e[1], np.int32) for e in exclusions if e is not None] or
                        [np.zeros(0, np.int32)]).astype(np.int32)
    if len(ei) == 0:
        ei = np.zeros(1, np.int32); ej = np.zeros(1, np.int32)
    return eo, ei, ej


def viterbi_search(ctx: Context, db: TargetDB, ids=None, exclusions=None, want_paths=True, hits=None,
                   paths=None):
    """One ViterbiRunner::alignment-style call with host buffers in and out.
    exclusions: optional list (per request) of (i_steps, j_steps) int arrays to mask (alt. alignments).
    hits/paths: optional caller-owned (e.g. pinned) output buffers."""
    ids = np.arange(db.n, dtype=np.int32) if ids is None else np.ascontiguousarray(ids, np.int32)
    n = len(ids)
    hits = np.zeros(n, HIT_DTYPE) if hits is None else hits
    cap = int(np.sum(ctx.Lq + db.Lh[np.clip(ids, 0, db.n - 1)].astype(np.int64) + 2))   # ids validated in C
    if want_paths and paths is None:
        paths = np.zeros(cap, np.uint8)
    if not want_paths:
        paths = None
    eo, ei, ej = _exclusions(exclusions)
    _ck(ctx.L.hhg_viterbi_search(ctx.h, db.h, n, _p(ids, c_i32p), hits.ctypes.data_as(C.c_void_p),
                                 _p(paths, c_u8p), cap if want_paths else 0, _p(eo, c_i64p), _p(ei, c_i32p),
                                 _p(ej, c_i32p)))
    return hits, paths


def query_set_batch(ctx: Context, queries, S33=None, q_pav=None, local=True, egq=0.0, egt=0.0, shift=-0.03, ssw=0.11,
                    use_ss=False, corr=0.1, ssm=2):
    """hhg_query_set_batch: queries = list of (p, tr[, ss]) prepared profiles; q_pav [nq, 20] for raw shards."""
    nq = len(queries)
    ps = [np.ascontiguousarray(q[0], np.float32) for q in queries]
    trs = [np.ascontiguousarray(q[1], np.float32) for q in queries]
    has_ss = all(len(q) > 2 and q[2] is not None for q in queries)
    sss = [np.ascontiguousarray(q[2], np.uint8) for q in queries] if has_ss else None
    Lq = np.array([p.shape[0] - 2 for p in ps], np.int32)
    pp = (C.c_void_p * nq)(*[p.ctypes.data for p in ps])
    tp = (C.c_void_p * nq)(*[t.ctypes.data for t in trs])
    sp = (C.c_void_p * nq)(*[x.ctypes.data for x in sss]) if has_ss else None
    S33 = None if S33 is None else np.ascontiguousarray(S33, np.float32)
    qv = None if q_pav is None else np.ascontiguousarray(q_pav, np.float32)
    par = Params(1 if local else 0, egq, egt, shift, ssw, 1 if use_ss else 0, corr, ssm)
    _ck(ctx.L.hhg_query_set_batch(ctx.h, nq, _p(Lq, c_i32p), pp, tp, sp, _p(qv, c_f32p), _p(S33, c_f32p), C.byref(par)))
    ctx.Lq = int(Lq[0])
    ctx.batch_Lq = Lq


def viterbi_search_batch(ctx: Context, db: TargetDB, req_query, ids, columnscore=1, pb=None, want_paths=True,
                         exclusions=None):
    """hhg_viterbi_search_batch: request k aligns query req_query[k] of the current batch with target ids[k].
    exclusions: optional list (per request) of (i_steps, j_steps) int arrays to mask, as in viterbi_search.
    columnscore 5 over a raw shard divides the named targets in the shard itself and leaves it unprepared (apply_null_model
    again before a single-query search); the queries must be divided by query_local_background."""
    rq = np.ascontiguousarray(req_query, np.int32); ids = np.ascontiguousarray(ids, np.int32)
    n = len(ids)
    hits = np.zeros(n, HIT_DTYPE)
    cap = int(np.sum(ctx.batch_Lq[np.clip(rq, 0, len(ctx.batch_Lq) - 1)].astype(np.int64) +
                     db.Lh[np.clip(ids, 0, db.n - 1)].astype(np.int64) + 2))
    paths = np.zeros(cap, np.uint8) if want_paths else None
    pbv = None if pb is None else np.ascontiguousarray(pb, np.float32)
    eo, ei, ej = _exclusions(exclusions)
    _ck(ctx.L.hhg_viterbi_search_batch(ctx.h, db.h, n, _p(rq, c_i32p), _p(ids, c_i32p), columnscore, _p(pbv, c_f32p),
                                       hits.ctypes.data_as(C.c_void_p), _p(paths, c_u8p), cap if want_paths else 0,
                                       _p(eo, c_i64p), _p(ei, c_i32p), _p(ej, c_i32p)))
    return hits, paths


def expand_path(hit, paths):
    """(i_steps, j_steps, states) arrays indexed 1..nsteps like Viterbi::BacktraceResult."""
    n = int(hit["nsteps"])
    st = paths[int(hit["path_off"]):int(hit["path_off"]) + n]
    i_s = np.zeros(n + 1, np.int32); j_s = np.zeros(n + 1, np.int32); s_s = np.zeros(n + 1, np.uint8)
    i, j = int(hit["i2"]), int(hit["j2"])
    # replay the walk: the recorded state at each step decides which index moved (src/hhviterbi.cpp:106-140);
    # the last recorded state was overwritten with MM, but positions do not depend on it.
    for k in range(n):
        i_s[k + 1], j_s[k + 1], s_s[k + 1] = i, j, st[k]
        s = st[k] if k < n - 1 else None
        if s == 2:
            i -= 1; j -= 1
        elif s in (3, 4):
            j -= 1
        elif s in (5, 6):
            i -= 1
    return i_s, j_s, s_s


def build_prefilter_profile(q_p, q_pav, lib219, offset=50, bit_factor=4):
    """Host-side query profile (stripe_query_profile, linear layout [220][Lq])."""
    q_p = np.ascontiguousarray(q_p, np.float32); q_pav = np.ascontiguousarray(q_pav, np.float32)
    lib219 = np.ascontiguousarray(lib219, np.float32)
    Lq = q_p.shape[0] - 2
    prof = np.zeros((220, Lq), np.uint8)
    _ck(load().hhg_prefilter_build_profile(Lq, _p(q_p, c_f32p), _p(q_pav, c_f32p), _p(lib219, c_f32p), offset,
                                           bit_factor, _p(prof, c_u8p)))
    return prof


def _profile_batch(profs):
    """(contiguous uint8 profiles, their lengths, the array of their addresses) as the batch prefilter calls take them;
    the profiles must stay referenced for the duration of the call."""
    profs = [np.ascontiguousarray(p, np.uint8) for p in profs]
    assert all(p.ndim == 2 and p.shape[0] == 220 for p in profs)
    Lq = np.array([p.shape[1] for p in profs], np.int32)
    return profs, Lq, (C.c_void_p * max(len(profs), 1))(*[p.ctypes.data for p in profs])


class CsDB:
    def __init__(self, ctx: Context, L, off, seq):
        self.ctx = ctx
        self.Lh = np.ascontiguousarray(L, np.int32)
        off = np.ascontiguousarray(off, np.int64); seq = np.ascontiguousarray(seq, np.uint8)
        h = C.c_void_p()
        _ck(ctx.L.hhg_csdb_create(ctx.h, len(self.Lh), _p(self.Lh, c_i32p), _p(off, c_i64p), _p(seq, c_u8p),
                                  C.byref(h)))
        self.h = h
        self.n = len(self.Lh)

    @classmethod
    def from_ffindex(cls, ctx, data: bytes, offsets, lengths):
        """The shard from <db>_cs219.ffdata + the (offset, length) columns of its .ffindex (init_prefilter)."""
        off = np.ascontiguousarray(offsets, np.int64); ln = np.ascontiguousarray(lengths, np.int64)
        h = C.c_void_p()
        buf = np.frombuffer(data, np.uint8)
        _ck(ctx.L.hhg_csdb_create_ffindex(ctx.h, len(off), buf.ctypes.data_as(C.c_char_p), _p(off, c_i64p), _p(ln, c_i64p),
                                          C.byref(h)))
        self = cls.__new__(cls)
        self.ctx, self.h, self.n = ctx, h, len(off)
        self.Lh = (ln - 1).astype(np.int32)
        return self

    def ungapped(self, prof, offset=50):
        prof = np.ascontiguousarray(prof, np.uint8)
        assert prof.shape[0] == 220
        sc = np.zeros(self.n, np.int32)
        _ck(self.ctx.L.hhg_prefilter_ungapped(self.ctx.h, self.h, prof.shape[1], _p(prof, c_u8p), offset,
                                              _p(sc, c_i32p)))
        return sc

    def sw(self, prof, ids=None, gap_open=24, gap_extend=4, bias=50):
        """Stage-2 gapped scores (swStripedByte) for the selected sequences."""
        prof = np.ascontiguousarray(prof, np.uint8)
        ids = None if ids is None else np.ascontiguousarray(ids, np.int32)
        n = self.n if ids is None else len(ids)
        sc = np.zeros(n, np.int32)
        _ck(self.ctx.L.hhg_prefilter_sw(self.ctx.h, self.h, n, _p(ids, c_i32p), prof.shape[1], _p(prof, c_u8p),
                                        gap_open, gap_extend, bias, _p(sc, c_i32p)))
        return sc

    def run(self, prof, offset=50, upload=True):
        prof = np.ascontiguousarray(prof, np.uint8)
        _ck(self.ctx.L.hhg_prefilter_ungapped_run(self.ctx.h, self.h, prof.shape[1], _p(prof, c_u8p), offset,
                                                  1 if upload else 0))

    def select(self, Lq, bit_factor=4, smax_thresh=10, min_hits=100):
        """Stage-1 selection on the device after run(): (ids, corrected scores) of the survivors in the reference's
        order (Prefilter::prefilter_db, src/hhprefilter.cpp:477-506)."""
        cap = self.n
        ids = np.zeros(cap, np.int32); sc = np.zeros(cap, np.int32); n = np.zeros(1, np.int32)
        _ck(self.ctx.L.hhg_prefilter_select(self.ctx.h, self.h, Lq, bit_factor, smax_thresh, min_hits, _p(ids, c_i32p),
                                            _p(sc, c_i32p), cap, _p(n, c_i32p)))
        return ids[:n[0]].copy(), sc[:n[0]].copy()

    def fetch(self):
        sc = np.zeros(self.n, np.int32)
        _ck(self.ctx.L.hhg_prefilter_fetch(self.ctx.h, self.h, _p(sc, c_i32p)))
        return sc

    # ---- query batches: each call equals the single-query call above made once per profile
    def max_batch(self) -> int:
        """Queries whose score rows fit the context's memory budget in one run_batch (at least 1)."""
        return int(self.ctx.L.hhg_prefilter_batch_max_queries(self.ctx.h, self.h))

    def run_batch(self, profs, offset=50):
        """hhg_prefilter_ungapped_batch_run: raw ungapped scores of every profile, left on the device."""
        profs, Lq, ptrs = _profile_batch(profs)
        _ck(self.ctx.L.hhg_prefilter_ungapped_batch_run(self.ctx.h, self.h, len(profs), _p(Lq, c_i32p), ptrs, offset))

    def fetch_batch(self, nq):
        """Raw scores of the last run_batch (nq profiles): [nq, n]."""
        sc = np.zeros((nq, self.n), np.int32)
        _ck(self.ctx.L.hhg_prefilter_ungapped_batch_fetch(self.ctx.h, self.h, _p(sc, c_i32p)))
        return sc

    def ungapped_batch(self, profs, offset=50):
        self.run_batch(profs, offset)
        return self.fetch_batch(len(profs))

    def select_batch(self, Lq, bit_factor=4, smax_thresh=10, min_hits=100, cap=None):
        """Stage-1 selection of every query of the last run_batch: one (ids, corrected scores) pair per query, each
        equal to select().  cap: total output capacity (default: every sequence for every query)."""
        Lq = np.ascontiguousarray(Lq, np.int32)
        nq = len(Lq)
        cap = nq * self.n if cap is None else int(cap)
        ids = np.empty(max(cap, 1), np.int32); sc = np.empty(max(cap, 1), np.int32); off = np.zeros(nq + 1, np.int32)
        _ck(self.ctx.L.hhg_prefilter_select_batch(self.ctx.h, self.h, nq, _p(Lq, c_i32p), bit_factor, smax_thresh,
                                                  min_hits, _p(ids, c_i32p), _p(sc, c_i32p), cap, _p(off, c_i32p)))
        return [(ids[off[q]:off[q + 1]].copy(), sc[off[q]:off[q + 1]].copy()) for q in range(nq)]

    def sw_batch(self, profs, req_query, ids, gap_open=24, gap_extend=4, bias=50):
        """Stage-2 gapped scores of request k = profile req_query[k] against sequence ids[k], in one launch."""
        profs, Lq, ptrs = _profile_batch(profs)
        rq = np.ascontiguousarray(req_query, np.int32); ids = np.ascontiguousarray(ids, np.int32)
        assert len(rq) == len(ids)
        sc = np.zeros(len(ids), np.int32)
        _ck(self.ctx.L.hhg_prefilter_sw_batch(self.ctx.h, self.h, len(profs), _p(Lq, c_i32p), ptrs, len(ids),
                                              _p(rq, c_i32p), _p(ids, c_i32p), gap_open, gap_extend, bias,
                                              _p(sc, c_i32p)))
        return sc

    def close(self):
        if self.h:
            self.ctx.L.hhg_csdb_destroy(self.h)
            self.h = None
