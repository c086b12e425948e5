"""The context-library pseudocounts of the query (hhg_context_library_create + hhg_query_context_pseudocounts: the
generative score in k_crf_scores on the device, the libm tail on the host) against the compiled reference, bit for bit
in p and pav: HH-suite's context_data.lib on seeded alignments of every shape family through the library's
alignment -> HMM step with both hhblits engines, every synthetic library under every admixture and window weight pair
(tests/golden/ctxlib_v1.npz), the lengths around the window up to the longest query (its reference in a child process),
one context alternating a CRF and a context library, and `-contxt context_data.lib` end to end into a search and into
the prefilter profile."""
import subprocess
import sys

import numpy as np
import pytest

from tests import crf_cases, msa_cases
from tests import ctxlib_cases as cc
from tests.test_msa_scale_gpu import _job, _reference, _write
from tests.util import ROOT, bits

pytestmark = pytest.mark.gpu

ENGINES = ((0, cc.ADMIX_HHM), (1, cc.ADMIX_PREFILTER))


def _cmp(got, want, tag):
    """p and pav bit for bit; on a difference name the first differing column and amino acid."""
    (p, pav), (rp, rpav) = got, want
    assert p.shape == rp.shape, (tag, p.shape, rp.shape)
    d = np.argwhere(bits(p) != bits(rp))
    assert len(d) == 0, (tag, f"{len(d)} entries differ, first at column {d[0][0]} amino acid {d[0][1]}",
                         float(p[tuple(d[0])]), float(rp[tuple(d[0])]))
    assert np.array_equal(bits(pav), bits(rpav)), (tag, "pav")


@pytest.fixture(scope="module")
def libref():
    from oracle.ctxlib_binding import LibRef
    try:
        return LibRef()
    except (FileNotFoundError, OSError) as e:
        pytest.skip(f"compiled reference not available: {e}")


@pytest.fixture(scope="module")
def shipped(hhg, gpu_ctx, libref):
    lib = hhg.capi.ContextLibrary(gpu_ctx, libref.lib_text())
    yield lib
    lib.close()


def _ref(libref, prof, engine):
    adm = ENGINES[engine][1]
    return libref.context_pc_lib(libref.lib_text(), cc.CSW, cc.CSB, *prof, *cc.admix_args(adm))


# ------------------------------------------------------------------------------------------- alignments of every family
SEEDS_PER_FAMILY = 16


@pytest.mark.parametrize("fam", msa_cases.FAMILIES)
def test_alignments_through_both_engines(hhg, gpu_ctx, refshim, libref, shipped, fam, tmp_path):
    """Seeded alignments: the library's hhg_msa_to_hmm then its library pseudocounts, against the reference's
    alignment -> HMM (in a child process) then its cs::LibraryPseudocounts, with both hhblits engines."""
    rng = np.random.default_rng([20261016, msa_cases.FAMILIES.index(fam)])
    texts = [msa_cases.random_alignment(rng, fam) for _ in range(SEEDS_PER_FAMILY)]
    pb = libref.pb()
    got = {}
    for k, t in enumerate(texts):
        try:
            got[k] = hhg.capi.msa_to_hmm(gpu_ctx, t, pb)
        except hhg.HhgError:
            pass                                # refused by the library: the reference would exit on it
    assert len(got) >= SEEDS_PER_FAMILY * 3 // 4, (fam, len(got))
    paths = _write(tmp_path, texts, "a")
    ok = sorted(got)
    refs = _reference([_job(paths[k]) for k in ok], tmp_path)
    for k, ref in zip(ok, refs):
        raw = got[k]
        for engine, adm in ENGINES:
            mine = shipped.pseudocounts(raw["f"], raw["neff_m"], raw["neff_hmm"], pb, hhg.capi.Admix(*adm))
            _cmp(mine, _ref(libref, (ref["f"], ref["neff_m"], ref["neff_hmm"]), engine), (fam, k, engine, paths[k]))


# ------------------------------------------------------------------------------------------------- synthetic libraries
@pytest.fixture(scope="module")
def G():
    with cc.golden() as z:
        yield z


@pytest.mark.parametrize("tag,text", cc.libraries(), ids=[t for t, _ in cc.libraries()])
def test_synthetic_libraries(hhg, gpu_ctx, G, tag, text):
    """Run-time K and W, ISLOG T and F: every admixture of the table with every window weight pair (reference: the
    goldens, which also hold the background pb)."""
    pb = G["pb"]
    cases = [c for c in cc.golden_cases() if c[0].startswith(f"lib/{tag}/")]
    assert len(cases) == len(cc.ADMIXTURES) * len(cc.WEIGHTS)
    libs = {wts: hhg.capi.ContextLibrary(gpu_ctx, text, *wts) for wts in cc.WEIGHTS}
    try:
        for key, t, wts, adm, prof in cases:
            p, pav = libs[wts].pseudocounts(*prof, pb, hhg.capi.Admix(*adm))
            cc.compare(p, pav, cc.expected(G, key, t, wts, adm, prof), key)
    finally:
        for lib in libs.values():
            lib.close()


# ------------------------------------------------------------------------------------------------------------ lengths
@pytest.mark.parametrize("L", [1, 13, 14, 1500])
def test_lengths(hhg, libref, shipped, L):
    """One column, the window, one past it and a long query, both engines, against the live reference."""
    prof = crf_cases.mixed(np.random.default_rng([L, 16]), L)
    for engine, adm in ENGINES:
        got = shipped.pseudocounts(*prof, libref.pb(), hhg.capi.Admix(*adm))
        _cmp(got, _ref(libref, prof, engine), (L, engine))


_CHILD = r"""
import sys
import numpy as np
sys.path.insert(0, sys.argv[1])
from oracle.ctxlib_binding import LibRef
from tests import crf_cases, ctxlib_cases as cc
L = int(sys.argv[2])
r = LibRef()
prof = crf_cases.longest_query(L)
out = {}
for engine, adm in ((0, cc.ADMIX_HHM), (1, cc.ADMIX_PREFILTER)):
    out[f"p{engine}"], out[f"pav{engine}"] = r.context_pc_lib(r.lib_text(), cc.CSW, cc.CSB, *prof, *cc.admix_args(adm))
np.savez(sys.argv[3], **out)
"""


def test_longest_query_equals_reference(hhg, libref, shipped, tmp_path):
    """L = 32 767, the query limit, against the reference run in a child process alongside the device."""
    L = crf_cases.MAX_QUERY
    script, out, log = tmp_path / "lib_child.py", tmp_path / "lib_long.npz", tmp_path / "lib_child.log"
    script.write_text(_CHILD)
    with open(log, "w") as lf:
        proc = subprocess.Popen([sys.executable, str(script), ROOT, str(L), str(out)], stdout=subprocess.DEVNULL, stderr=lf)
        prof = crf_cases.longest_query(L)
        got = [shipped.pseudocounts(*prof, libref.pb(), hhg.capi.Admix(*adm)) for _, adm in ENGINES]
        rc = proc.wait()
    assert rc == 0, f"the compiled reference failed with exit code {rc}: {log.read_text()[-2000:]}"
    with np.load(out) as z:
        for engine, _ in ENGINES:
            _cmp(got[engine], (z[f"p{engine}"], z[f"pav{engine}"]), ("L = 32767", engine))


def test_refusals_launch_nothing(hhg, gpu_ctx, libref, shipped):
    """A text the reader refuses and a query over the limit are refused before anything is allocated or launched."""
    n0 = gpu_ctx.launches
    for _, text, msg in cc.refused_by_library():
        with pytest.raises(hhg.HhgError, match=msg):
            hhg.capi.ContextLibrary(gpu_ctx, text)
    L = crf_cases.MAX_QUERY + 1
    f = np.full((L + 2, 20), 0.05, np.float32); neff_m = np.ones(L + 1, np.float32)
    with pytest.raises(hhg.HhgError, match="query limit of 32767"):
        shipped.pseudocounts(f, neff_m, 1.0, libref.pb(), hhg.capi.Admix(*cc.ADMIX_HHM))
    assert gpu_ctx.launches == n0


# --------------------------------------------------------------------------------------------------- context reuse
def test_one_context_crf_and_library(hhg, refshim, libref):
    """One context, the shipped CRF (query-HMM admixture) and the shipped context library (prefilter admixture)
    alternating over five lengths, sharing the grow-only staging: every result equals the reference."""
    ctx = hhg.Context()
    crf = hhg.capi.Crf(ctx, refshim.crf_text())
    lib = hhg.capi.ContextLibrary(ctx, libref.lib_text())
    profiles = crf_cases.reuse_profiles()
    try:
        for rnd in range(2):
            for k, L in enumerate(crf_cases.REUSE_LENGTHS):
                prof = profiles[L]
                if (k + rnd) % 2 == 0:
                    got = crf.pseudocounts(*prof, refshim.pb(), hhg.capi.Admix(*cc.ADMIX_HHM))
                    _cmp(got, refshim.context_pc(*prof, engine=0), (rnd, L, "crf"))
                else:
                    got = lib.pseudocounts(*prof, libref.pb(), hhg.capi.Admix(*cc.ADMIX_PREFILTER))
                    _cmp(got, _ref(libref, prof, 1), (rnd, L, "library"))
    finally:
        crf.close(); lib.close(); ctx.close()


# ----------------------------------------------------------------------------------------- -contxt context_data.lib
def test_contxt_lib_query_path_end_to_end(hhg, gpu_ctx, refshim, oracle, libref, shipped, tmp_path):
    """hhblits -contxt context_data.lib on query.a3m: the library's alignment -> HMM -> library pseudocounts (engine 0)
    -> hhg_query_set -> viterbi_search over a small shard equals the oracle's Viterbi on the arrays the reference
    prepared; engine 1 -> hhg_prefilter_build_profile equals the reference's stripe_query_profile of its own profile.
    One background throughout, the one the reference's alignment reader holds."""
    default_pb = libref.pb()
    libref.set_pb(refshim.pb())
    try:
        _contxt_lib_query_path(hhg, gpu_ctx, refshim, oracle, libref, shipped, tmp_path)
    finally:
        libref.set_pb(default_pb)


def _contxt_lib_query_path(hhg, gpu_ctx, refshim, oracle, libref, shipped, tmp_path):
    qa = msa_cases.texts()[-1]
    qpath = tmp_path / "q.a3m"
    qpath.write_bytes(qa)
    pb, R = refshim.pb(), refshim.R()
    raw = hhg.capi.msa_to_hmm(gpu_ctx, qa, pb)
    p0, pav0 = shipped.pseudocounts(raw["f"], raw["neff_m"], raw["neff_hmm"], pb, hhg.capi.Admix(*cc.ADMIX_HHM))
    q = hhg.capi.query_from_a3m(gpu_ctx, qa, R, pb)
    ref = refshim.msa_to_hmm(str(qpath), prep=True)
    ref_p0, ref_pav0 = _ref(libref, (ref["f"], ref["neff_m"], ref["neff_hmm"]), 0)
    _cmp((p0, pav0), (ref_p0, ref_pav0), "engine 0")
    assert np.array_equal(bits(q["tr"]), bits(ref["tr_prep"]))
    texts = msa_cases.texts()[:6]
    gpu_ctx.set_query(p0, q["tr"])
    data = b"".join(t + b"\0" for t in texts)
    ln = np.array([len(t) + 1 for t in texts], np.int64)
    off = np.concatenate([[0], np.cumsum(ln)[:-1]]).astype(np.int64)
    db = hhg.TargetDB.from_a3m(gpu_ctx, data, off, ln, R, pb)
    db.apply_null_model(q_pav=pav0, pb=pb, columnscore=1)
    hits, paths = hhg.viterbi_search(gpu_ctx, db)
    db.close()
    for k, t in enumerate(texts):
        tp = tmp_path / f"t{k}.a3m"
        tp.write_bytes(t)
        tref = refshim.msa_to_hmm(str(tp), prep=True)
        pnul = (0.5 * (ref_pav0.astype(np.float32) + tref["pav"])).astype(np.float32)
        t_p = tref["p"].copy()
        t_p[1:tref["L"] + 1] = (t_p[1:tref["L"] + 1] / pnul).astype(np.float32)
        sc, i2, j2, bt = oracle.viterbi(ref_p0, ref["tr_prep"], t_p, tref["tr_prep"])
        h = hits[k]
        assert bits(h["score"]) == bits(sc) and (h["i2"], h["j2"]) == (i2, j2), k
        n, _, _, st, mc = oracle.backtrace(bt, i2, j2)
        assert h["nsteps"] == n and h["matched_cols"] == mc, k
        assert np.array_equal(paths[h["path_off"]:h["path_off"] + n], st[1:]), k
    p1, pav1 = shipped.pseudocounts(raw["f"], raw["neff_m"], raw["neff_hmm"], pb, hhg.capi.Admix(*cc.ADMIX_PREFILTER))
    ref_p1, ref_pav1 = _ref(libref, (ref["f"], ref["neff_m"], ref["neff_hmm"]), 1)
    _cmp((p1, pav1), (ref_p1, ref_pav1), "engine 1")
    prof = hhg.capi.build_prefilter_profile(p1, pav1, refshim.cs219(), 50, 4)
    refshim.set_query(ref_p1, ref["tr_prep"], ref_pav1)
    qc, W = refshim.stripe_query_profile(50, 4)
    pos = np.arange(ref["L"])
    want = np.stack([qc[a * W * 32 + (pos % W) * 32 + pos // W] for a in range(220)])
    assert np.array_equal(prof, want)
