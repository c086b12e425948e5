"""The context-specific (CRF) pseudocounts of the query (hhg_crf_create + hhg_query_context_pseudocounts: k_crf_scores on
the device, the libm tail on the host) at the shapes where they can go wrong, against the compiled reference run on the
same host, bit for bit in p and pav: every count-profile family of tests/crf_cases.py with both default engines, every
admixture of the table, synthetic libraries of 1..1000 states and windows of 1..63 columns, seeded alignments of every
shape family through the library's alignment -> HMM step, the longest query (32 767 columns, its reference in a child
process), one context switching libraries and lengths, and the default hhblits query path into a search and into the
prefilter profile.  The two default engines on the embedded library are compared with the compiled reference run on the
same host; custom libraries and the other admixtures with tests/golden/crf_v1.npz, which that reference made
(tests/crf_cases.py explains why)."""
import os
import subprocess
import sys

import numpy as np
import pytest

from tests import crf_cases, msa_cases
from tests.test_msa_scale_gpu import _job, _reference, _write
from tests.util import ROOT, bits

pytestmark = pytest.mark.gpu

ENGINES = ((0, crf_cases.ADMIX_HHM), (1, crf_cases.ADMIX_PREFILTER))


def _cmp(got, want, tag):
    """p and pav bit for bit; on a difference name the first differing column and amino acid."""
    (p, pav), (rp, rpav) = got, want
    assert p.shape == rp.shape, (tag, p.shape, rp.shape)
    d = np.argwhere(bits(p) != bits(rp))
    assert len(d) == 0, (tag, f"{len(d)} entries differ, first at column {d[0][0]} amino acid {d[0][1]}",
                         float(p[tuple(d[0])]), float(rp[tuple(d[0])]))
    assert rpav is None or np.array_equal(bits(pav), bits(rpav)), (tag, "pav")


@pytest.fixture(scope="module")
def embedded(hhg, gpu_ctx, refshim):
    crf = hhg.capi.Crf(gpu_ctx, refshim.crf_text())
    yield crf
    crf.close()


def _admix(hhg, adm):
    return hhg.capi.Admix(*adm)


# ------------------------------------------------------------------------------------------ count profiles, default engines
@pytest.mark.parametrize("fam", crf_cases.FAMILIES)
def test_count_profile_families(hhg, refshim, embedded, fam):
    """Each family with the embedded 4000-state, 13-column library and both default engines (query HMM: HHsearch
    0.9 / 4.0 / 1.0, prefilter: CS-BLAST 0.8 / 2.0)."""
    pb = refshim.pb()
    for tag, (f, neff_m, neff_hmm) in crf_cases.family(fam):
        for engine, adm in ENGINES:
            got = embedded.pseudocounts(f, neff_m, neff_hmm, pb, _admix(hhg, adm))
            _cmp(got, refshim.context_pc(f, neff_m, neff_hmm, engine=engine), (tag, engine))


@pytest.fixture(scope="module")
def G():
    with crf_cases.golden() as z:
        yield z


@pytest.fixture(scope="module")
def golden_cases(refshim):
    return crf_cases.golden_cases(refshim.crf_text())


@pytest.mark.parametrize("ai", range(len(crf_cases.ADMIXTURES)), ids=[str(a) for a in crf_cases.ADMIXTURES])
def test_admixture_table(hhg, refshim, embedded, G, golden_cases, ai):
    """Every admixture of the table on the edge, single-sequence and diverse families (reference: the goldens)."""
    pb = refshim.pb()
    cases = [c for c in golden_cases["admix"] if c[0].startswith(f"admix/{ai}/")]
    assert len(cases) == len(crf_cases.family("edges")) + 5 + 3
    for key, text, adm, (f, neff_m, neff_hmm) in cases:
        p, pav = embedded.pseudocounts(f, neff_m, neff_hmm, pb, _admix(hhg, adm))
        crf_cases.compare(p, pav, crf_cases.expected(G, key, text, adm, (f, neff_m, neff_hmm)), key)


@pytest.mark.parametrize("tag,text", crf_cases.libraries(), ids=[t for t, _ in crf_cases.libraries()])
def test_synthetic_libraries(hhg, gpu_ctx, refshim, G, golden_cases, tag, text):
    """Run-time K and W: the edge family relative to the library's window and a 400-column diverse profile, the two
    default admixtures alternating (reference: the goldens)."""
    crf = hhg.capi.Crf(gpu_ctx, text)
    pb = refshim.pb()
    cases = [c for c in golden_cases["lib"] if c[0].startswith(f"lib/{tag}/")]
    assert len(cases) == len(crf_cases.family("edges", W=crf.window)) + 1
    for key, t, adm, (f, neff_m, neff_hmm) in cases:
        p, pav = crf.pseudocounts(f, neff_m, neff_hmm, pb, _admix(hhg, adm))
        crf_cases.compare(p, pav, crf_cases.expected(G, key, t, adm, (f, neff_m, neff_hmm)), key)
    crf.close()


# ------------------------------------------------------------------------------------------- alignments of every family
SEEDS_PER_FAMILY = 16


@pytest.mark.parametrize("fam", msa_cases.FAMILIES)
def test_alignments_through_both_pipelines(hhg, gpu_ctx, refshim, embedded, fam, tmp_path):
    """Seeded alignments: the library's hhg_msa_to_hmm then its pseudocounts, against the reference's alignment -> HMM
    (in a child process) then its context_pc, with both default engines."""
    rng = np.random.default_rng([20261015, msa_cases.FAMILIES.index(fam)])
    texts = [msa_cases.random_alignment(rng, fam) for _ in range(SEEDS_PER_FAMILY)]
    pb = refshim.pb()
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
            mine = embedded.pseudocounts(raw["f"], raw["neff_m"], raw["neff_hmm"], pb, _admix(hhg, adm))
            want = refshim.context_pc(ref["f"], ref["neff_m"], ref["neff_hmm"], engine=engine)
            _cmp(mine, want, (fam, k, engine, paths[k]))


# ------------------------------------------------------------------------------------------------------- query limit
_CHILD = r"""
import sys
import numpy as np
sys.path.insert(0, sys.argv[1])
from oracle.binding import RefShim
from tests import crf_cases
L = int(sys.argv[2])
r = RefShim(nocontxt=True, maxres=L + 2)
f, neff_m, neff_hmm = crf_cases.longest_query(L)
out = {}
for engine in (0, 1):
    out[f"p{engine}"], out[f"pav{engine}"] = r.context_pc(f, neff_m, neff_hmm, engine=engine)
np.savez(sys.argv[3], **out)
"""


def test_longest_query_equals_reference(hhg, gpu_ctx, refshim, embedded, tmp_path):
    """L = 32 767, the query limit: 32 767 block rows of k_crf_scores and 1 GiB of device and pinned staging.  The
    reference needs maxres = L + 2, so it runs in a child process."""
    L = crf_cases.MAX_QUERY
    script, out = tmp_path / "crf_child.py", tmp_path / "crf_long.npz"
    script.write_text(_CHILD)
    log = tmp_path / "crf_child.log"
    with open(log, "w") as lf:
        proc = subprocess.Popen([sys.executable, str(script), ROOT, str(L), str(out)], stdout=subprocess.DEVNULL, stderr=lf)
        f, neff_m, neff_hmm = crf_cases.longest_query(L)
        pb = refshim.pb()
        got = [embedded.pseudocounts(f, neff_m, neff_hmm, pb, _admix(hhg, adm)) for _, adm in ENGINES]
        rc = proc.wait()
    assert rc == 0, f"the compiled reference failed with exit code {rc}: {log.read_text()[-2000:]}"
    with np.load(out) as z:
        for engine, _ in ENGINES:
            _cmp(got[engine], (z[f"p{engine}"], z[f"pav{engine}"]), ("L = 32767", engine))


def test_query_longer_than_limit_is_refused(hhg, gpu_ctx, embedded, refshim):
    """L = 32 768 is refused with a message naming the query limit, before anything is allocated or launched."""
    L = crf_cases.MAX_QUERY + 1
    f = np.full((L + 2, 20), 0.05, np.float32); neff_m = np.ones(L + 1, np.float32)
    n0 = gpu_ctx.launches
    with pytest.raises(hhg.HhgError, match="query limit of 32767"):
        embedded.pseudocounts(f, neff_m, 1.0, refshim.pb(), _admix(hhg, crf_cases.ADMIX_HHM))
    assert gpu_ctx.launches == n0


def test_crf_from_another_device_is_refused(hhg, refshim):
    """A library uploaded on device 1 used with a context on device 0: refused before anything is launched, since the
    kernel would read the other device's memory."""
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    ctx0, ctx1 = hhg.Context(device=0), hhg.Context(device=1)
    crf = hhg.capi.Crf(ctx1, crf_cases.library(2, 3))
    try:
        f, neff_m, neff_hmm = crf_cases.edge_profile(np.random.default_rng(0), 20)
        crf.ctx = ctx0
        n0 = ctx0.launches
        with pytest.raises(hhg.HhgError, match="device 1, the context is on device 0"):
            crf.pseudocounts(f, neff_m, neff_hmm, refshim.pb(), _admix(hhg, crf_cases.ADMIX_HHM))
        assert ctx0.launches == n0
        crf.ctx = ctx1
        p, _ = crf.pseudocounts(f, neff_m, neff_hmm, refshim.pb(), _admix(hhg, crf_cases.ADMIX_HHM))
        assert np.all(np.isfinite(p))
    finally:
        crf.close(); ctx0.close(); ctx1.close()


# --------------------------------------------------------------------------------------------------- context reuse
def test_one_context_two_libraries(hhg, refshim, G, golden_cases):
    """One context, the embedded 4000 x 13 library (query-HMM admixture, against the live reference) and a synthetic
    257 x 63 one (prefilter admixture, against the goldens) alternating, while L goes 400 -> 4094 -> 1 -> 13 -> 2000
    (the grow-only staging buffers are shared across both): every result equals the reference, a repeated call is
    bit-identical, and a call without pav leaves rows 1..L unchanged."""
    ctx = hhg.Context()
    embedded_text = refshim.crf_text()
    crfs = [hhg.capi.Crf(ctx, embedded_text), hhg.capi.Crf(ctx, crf_cases.library(*crf_cases.SYNTH_REUSE))]
    synth = {int(key.split("=")[1]): (key, text, adm) for key, text, adm, _ in golden_cases["reuse"]}
    pb = refshim.pb()
    profiles = crf_cases.reuse_profiles()
    first = None
    try:
        for rnd in range(2):
            for k, L in enumerate(crf_cases.REUSE_LENGTHS):
                which = (k + rnd) % 2
                f, neff_m, neff_hmm = profiles[L]
                if which == 0:
                    got = crfs[0].pseudocounts(f, neff_m, neff_hmm, pb, _admix(hhg, crf_cases.ADMIX_HHM))
                    _cmp(got, refshim.context_pc(f, neff_m, neff_hmm, engine=0), (rnd, L, "embedded"))
                else:
                    key, text, adm = synth[L]
                    got = crfs[1].pseudocounts(f, neff_m, neff_hmm, pb, _admix(hhg, adm))
                    crf_cases.compare(*got, crf_cases.expected(G, key, text, adm, profiles[L]), (rnd, key))
                first = first or (L, which, got)
        L, which, (p, pav) = first
        f, neff_m, neff_hmm = profiles[L]
        adm = (crf_cases.ADMIX_HHM, crf_cases.ADMIX_PREFILTER)[which]
        again = crfs[which].pseudocounts(f, neff_m, neff_hmm, pb, _admix(hhg, adm))
        assert again[0].tobytes() == p.tobytes() and again[1].tobytes() == pav.tobytes()
        p2, none = crfs[which].pseudocounts(f, neff_m, neff_hmm, pb, _admix(hhg, adm), want_pav=False)
        assert none is None and p2[1:L + 1].tobytes() == p[1:L + 1].tobytes()
    finally:
        for c in crfs:
            c.close()
        ctx.close()


# ------------------------------------------------------------------------------------------ default hhblits query path
def _queries():
    from hhsuite_b200 import synth
    return [("single sequence", synth.a3m_text(150, 0, 42).encode()), ("query.a3m", msa_cases.texts()[-1])]


@pytest.mark.parametrize("which", [0, 1], ids=["single_sequence", "query_a3m"])
def test_default_hhblits_query_path_end_to_end(hhg, gpu_ctx, refshim, oracle, embedded, which, tmp_path):
    """The library's query alignment -> HMM -> engine-0 pseudocounts + query_from_a3m transitions -> hhg_query_set ->
    viterbi_search over a small shard equals the oracle's Viterbi on the arrays the reference prepared: score bits, end
    cells and paths.  Engine 1 -> hhg_prefilter_build_profile equals the reference's stripe_query_profile of its own
    engine-1 profile."""
    tag, qa = _queries()[which]
    qpath = tmp_path / "q.a3m"
    qpath.write_bytes(qa)
    pb, R = refshim.pb(), refshim.R()
    raw = hhg.capi.msa_to_hmm(gpu_ctx, qa, pb)
    p0, pav0 = embedded.pseudocounts(raw["f"], raw["neff_m"], raw["neff_hmm"], pb, _admix(hhg, crf_cases.ADMIX_HHM))
    q = hhg.capi.query_from_a3m(gpu_ctx, qa, R, pb)
    ref = refshim.msa_to_hmm(str(qpath), prep=True)
    ref_p0, ref_pav0 = refshim.context_pc(ref["f"], ref["neff_m"], ref["neff_hmm"], engine=0)
    _cmp((p0, pav0), (ref_p0, ref_pav0), (tag, "engine 0"))
    assert np.array_equal(bits(q["tr"]), bits(ref["tr_prep"])), tag
    # search: the library end to end against the oracle on the reference's arrays
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
        assert bits(h["score"]) == bits(sc) and (h["i2"], h["j2"]) == (i2, j2), (tag, k)
        n, _, _, st, mc = oracle.backtrace(bt, i2, j2)
        assert h["nsteps"] == n and h["matched_cols"] == mc, (tag, k)
        assert np.array_equal(paths[h["path_off"]:h["path_off"] + n], st[1:]), (tag, k)
    # prefilter profile: engine 1
    p1, pav1 = embedded.pseudocounts(raw["f"], raw["neff_m"], raw["neff_hmm"], pb, _admix(hhg, crf_cases.ADMIX_PREFILTER))
    ref_p1, ref_pav1 = refshim.context_pc(ref["f"], ref["neff_m"], ref["neff_hmm"], engine=1)
    _cmp((p1, pav1), (ref_p1, ref_pav1), (tag, "engine 1"))
    prof = hhg.capi.build_prefilter_profile(p1, pav1, refshim.cs219(), 50, 4)
    refshim.set_query(ref_p1, ref["tr_prep"], ref_pav1)
    qc, W = refshim.stripe_query_profile(50, 4)
    pos = np.arange(ref["L"])
    want = np.stack([qc[a * W * 32 + (pos % W) * 32 + pos // W] for a in range(220)])
    assert np.array_equal(prof, want), tag
