"""The alignment -> HMM kernels (k_msa_filter / _weights / _mstate / _finish) and the group loop of the database loaders
at database scale, against the compiled reference run on the same host, bit for bit: seeded random alignments of every
shape family of tests/msa_cases.py under all three match-state rules, one database of mixed shapes loaded at several
group sizes, repeated loads, a compressed database, and the record named by a load error.

The reference calls exit() on some inputs, so it only sees records the library's scanner accepted, and it runs in
child processes that write .npz files: an exit then fails one test, and the inputs stay under its tmp_path."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

from tests import msa_cases
from tests.test_hhm_db_gpu import _expected_records
from tests.test_msa_gpu import _cmp, _pack
from tests.util import ROOT, bits

pytestmark = pytest.mark.gpu

DEFAULT_PC = (2, 1.0, 1.5, 1.0)
HOST_TAU_PC = (2, 0.9, 4.0, 0.7)          # pcm 2 with pcc != 1: the loader computes tau per column on the host
DEGENERATE = ("master_only", "short_window", "identical", "long_inserts")

_CHILD = r"""
import json, sys
import numpy as np
sys.path.insert(0, sys.argv[1])
from oracle.binding import RefShim
r = RefShim(nocontxt=True, maxres=4096)
out = {}
for i, j in json.load(open(sys.argv[2])):
    sys.stderr.write(f"job {i}\n"); sys.stderr.flush()
    r.set_M(j["M"], j["Mgaps"]); r.set_pc(*j["pc"])
    kw = dict(filt=j["filt"], wg=j["wg"], prep=j["prep"])
    d = r.ca3m_to_hmm(j["path"], j["name"], **kw) if j.get("name") else r.msa_to_hmm(j["path"], **kw)
    for k, v in d.items():
        if k not in ("X", "I", "nres", "ksort"):
            out[f"{i}/{k}"] = np.asarray(v)
np.savez(sys.argv[3], **out)
"""


def _job(path, M=1, Mgaps=50, filt=None, wg=0, prep=False, pc=DEFAULT_PC, name=None):
    return dict(path=str(path), M=M, Mgaps=Mgaps, filt=None if filt is None else list(filt), wg=wg, prep=prep,
                pc=list(pc), name=name)


def _reference(jobs, directory):
    """The compiled reference on every job (msa_to_hmm, or ca3m_to_hmm when the job names an entry), in up to eight
    child processes; returns one result dict per job."""
    directory = str(directory)
    script = os.path.join(directory, "ref_child.py")
    with open(script, "w") as f:
        f.write(_CHILD)
    P = max(1, min(8, os.cpu_count() or 1, len(jobs)))
    procs = []
    for p in range(P):
        part = [(i, jobs[i]) for i in range(p, len(jobs), P)]
        jf, of, ef = (os.path.join(directory, f"ref_{p}.{x}") for x in ("json", "npz", "log"))
        with open(jf, "w") as f:
            json.dump(part, f)
        log = open(ef, "w")
        procs.append((subprocess.Popen([sys.executable, script, ROOT, jf, of], stderr=log, stdout=subprocess.DEVNULL), log, of, ef))
    out = [dict() for _ in jobs]
    failed = []
    for proc, log, of, ef in procs:
        rc = proc.wait()
        log.close()
        if rc != 0:
            lines = open(ef).read().splitlines()
            last = [ln for ln in lines if ln.startswith("job ")]
            failed.append((rc, jobs[int(last[-1].split()[1])] if last else None, lines[-3:]))
            continue
        with np.load(of) as z:
            for key in z.files:
                i, k = key.split("/")
                v = z[key]
                out[int(i)][k] = v.item() if v.ndim == 0 else v
    assert not failed, f"the compiled reference failed (exit code, input, last lines of its log): {failed}"
    return out


def _write(directory, texts, stem):
    paths = []
    for k, t in enumerate(texts):
        paths.append(os.path.join(str(directory), f"{stem}{k:04d}.a3m"))
        with open(paths[-1], "wb") as f:
            f.write(t)
    return paths


def _prep_params(hhg, refshim, pc):
    pp = refshim.prep_params()
    return hhg.capi.PrepParams(pp.gapb, pp.gapd, pp.gape, pp.gapf, pp.gapg, pp.gaph, pp.gapi, *pc)


def _expected_shard(refs):
    """Column records and pav of a shard whose records the reference prepared (prep=True results, in record order)."""
    want = np.concatenate([_expected_records(r["p"], r["tr_prep"], (r["ss_pred"].astype(np.int32) * 11 + r["ss_conf"]).astype(np.uint8),
                                             True) for r in refs])
    return want, np.stack([r["pav"] for r in refs]), np.array([r["L"] for r in refs], np.int32)


def _check_shard(db, expected, tag):
    want, pav_want, L = expected
    cols, pav = db.read_cols(0), db.read_pav()
    assert np.array_equal(db.Lh, L), (tag, "lengths")
    cb = np.flatnonzero((cols.view(np.uint32).reshape(len(cols), -1) != want.view(np.uint32).reshape(len(want), -1)).any(axis=1))
    assert len(cb) == 0, (tag, "column records differ in records", np.unique(np.searchsorted(np.cumsum(L), cb, side="right"))[:8].tolist())
    kb = np.flatnonzero((bits(pav) != bits(pav_want)).any(axis=1))
    assert len(kb) == 0, (tag, "pav differs for records", kb[:8].tolist())
    return cols, pav


def _load(hhg, ctx, texts, refshim, pc=DEFAULT_PC, group=None, monkeypatch=None):
    if group is None:
        monkeypatch.delenv("HHG_MSA_CHUNK_RECORDS", raising=False)
    else:
        monkeypatch.setenv("HHG_MSA_CHUNK_RECORDS", str(group))
    data, off, ln = _pack(texts)
    try:
        return hhg.TargetDB.from_a3m(ctx, data, off, ln, refshim.R(), refshim.pb(), params=_prep_params(hhg, refshim, pc))
    finally:
        monkeypatch.delenv("HHG_MSA_CHUNK_RECORDS", raising=False)


# ------------------------------------------------------------------------------------------------ random single alignments
def _single_specs(rng):
    """About 300 (kind, M, Mgaps): the A3M families under M = 1, aligned FASTA under -M 50 / -M 25 / -M first.  The
    largest families come first, then a shuffled mix, so one context sees sizes go down and up many times."""
    rest = (["typical"] * 90 + ["tiny"] * 70 + [f for f in DEGENERATE for _ in range(10)] + ["long"] * 7 + ["deep"] * 4)
    specs = [(f, 1, 50) for f in rest] + [("fasta", M, Mg) for (M, Mg) in ((2, 50), (2, 25), (3, 50)) for _ in range(30)]
    order = rng.permutation(len(specs))
    return [("long", 1, 50), ("deep", 1, 50)] + [specs[i] for i in order]


def test_random_alignments_equal_compiled_reference(hhg, gpu_ctx, refshim, tmp_path):
    """hhg_msa_to_hmm on one context, alignment after alignment, with random filter options and weighting mode."""
    rng = np.random.default_rng(20261015)
    pb, S = refshim.pb(), refshim.S()
    cases = []
    for k, (kind, M, Mg) in enumerate(_single_specs(rng)):
        t = msa_cases.random_fasta(rng, M, Mg) if kind == "fasta" else msa_cases.random_alignment(rng, kind)
        filt, wg = msa_cases.random_filter(rng)
        cases.append((k, kind, M, Mg, filt, wg, t))
    paths = _write(tmp_path, [c[-1] for c in cases], "s")
    got, refused = {}, []
    for (k, kind, M, Mg, filt, wg, t) in cases:
        mp = hhg.capi.MsaParams.defaults(M=M, Mgaps=Mg, max_seqid=filt[0], coverage=filt[1], qid=filt[2], qsc=filt[3],
                                         Ndiff=filt[4], wg=wg)
        try:
            got[k] = hhg.capi.msa_to_hmm(gpu_ctx, t, pb, S=S, mp=mp)
        except hhg.HhgError as e:
            refused.append((k, str(e)))
    # the kernels refuse what makes the reference exit (no row left after filtering, a zero divisor of the identity
    # schedule); such inputs must not reach the reference of the other cases, so each one runs alone
    for k, msg in refused:
        _, kind, M, Mg, filt, wg, _ = cases[k]
        with pytest.raises(AssertionError, match="the compiled reference failed"):
            _reference([_job(paths[k], M, Mg, filt, wg)], tmp_path / f"refused{k}")
    assert len(refused) <= len(cases) // 20, refused
    ok = [c for c in cases if c[0] in got]
    refs = _reference([_job(paths[k], M, Mg, filt, wg) for (k, kind, M, Mg, filt, wg, _) in ok], tmp_path)
    for (k, kind, M, Mg, filt, wg, _), ref in zip(ok, refs):
        _cmp(got[k], ref, f"alignment {k} ({kind}, M={M}/{Mg}, filter {filt}, wg={wg}, {paths[k]})")
    kinds = {c[1] for c in ok}
    assert kinds >= set(msa_cases.FAMILIES) | {"fasta"}, kinds


# ------------------------------------------------------------------------------------------ one database of mixed shapes
@pytest.fixture(scope="module")
def mixed(refshim, tmp_path_factory):
    """600 records of every family in shuffled order, and the reference's prepared HMM of each for both pseudocount
    settings."""
    d = tmp_path_factory.mktemp("mixed")
    rng = np.random.default_rng(600)
    fams = ["tiny"] * 150 + ["typical"] * 340 + ["long"] * 30 + ["deep"] * 12 + [f for f in DEGENERATE for _ in range(17)]
    fams = [fams[i] for i in rng.permutation(len(fams))]
    texts = [msa_cases.random_alignment(rng, f) for f in fams]
    paths = _write(d, texts, "m")
    refs = _reference([_job(p, prep=True, pc=pc) for pc in (DEFAULT_PC, HOST_TAU_PC) for p in paths], d)
    n = len(texts)
    return dict(texts=texts, families=fams, expected={DEFAULT_PC: _expected_shard(refs[:n]), HOST_TAU_PC: _expected_shard(refs[n:])})


@pytest.mark.parametrize("pc", [DEFAULT_PC, HOST_TAU_PC])
def test_mixed_database_at_every_group_size(hhg, gpu_ctx, refshim, mixed, pc, monkeypatch):
    """hhg_db_create_a3m in one group, and in groups of 1, 7 and 61 records: tiny and 3 000-column alignments share
    groups (and k_msa_mstate's queue), grow-only buffers are reused from group to group, the pieces are assembled."""
    assert len(mixed["texts"]) == 600 and set(mixed["families"]) == set(msa_cases.FAMILIES)
    shards = []
    for group in (None, 1, 7, 61):
        db = _load(hhg, gpu_ctx, mixed["texts"], refshim, pc, group, monkeypatch)
        cols, pav = _check_shard(db, mixed["expected"][pc], f"group size {group or 'all'}, pseudocounts {pc}")
        shards.append(cols.tobytes() + pav.tobytes())
        db.close()
    assert all(s == shards[0] for s in shards[1:])


def test_repeated_loads_are_byte_identical(hhg, gpu_ctx, refshim, mixed, monkeypatch):
    """Which block takes which (alignment, column) item changes from run to run; the shard must not."""
    out = []
    ctx2 = hhg.Context()
    try:
        for ctx in (gpu_ctx, gpu_ctx, ctx2):
            db = _load(hhg, ctx, mixed["texts"], refshim, monkeypatch=monkeypatch)
            out.append((db.read_cols(0).tobytes(), db.read_pav().tobytes()))
            db.close()
    finally:
        ctx2.close()
    assert out[1] == out[0] and out[2] == out[0]


def test_error_names_the_record_then_context_loads(hhg, gpu_ctx, refshim, mixed, monkeypatch):
    """A record the reader refuses (a dropped '>aa_' header followed by another sequence) at position 437 of 600: the
    load fails naming that record, in one group and in groups of 61, and the context then loads a correct shard."""
    texts = list(mixed["texts"])
    texts[437] += b">aa_dropped\nACDEFGHIKL\n>after\nACDEFGHIKL\n"
    assert not msa_cases.accepted(texts[437]) and msa_cases.accepted(mixed["texts"][437])
    for group in (None, 61):
        with pytest.raises(hhg.HhgError, match=r"record 437\b"):
            _load(hhg, gpu_ctx, texts, refshim, group=group, monkeypatch=monkeypatch)
    db = _load(hhg, gpu_ctx, mixed["texts"], refshim, group=61, monkeypatch=monkeypatch)
    _check_shard(db, mixed["expected"][DEFAULT_PC], "after a failed load")
    db.close()


# ----------------------------------------------------------------------------------------------- compressed database
def test_compressed_database_at_scale(hhg, gpu_ctx, refshim, tmp_path):
    """150 records through synth.a3m_to_ca3m: hhg_ca3m_to_hmm one by one and hhg_db_create_ca3m at once."""
    from hhsuite_b200 import ffindex
    rng = np.random.default_rng(150)
    fams = ["tiny"] * 40 + ["typical"] * 90 + ["long"] * 4 + ["deep"] * 2 + [f for f in DEGENERATE for _ in range(4)]
    fams = [fams[i] for i in rng.permutation(len(fams))]
    prefix = msa_cases.ca3m_database(tmp_path, [(f"al{k:04d}", msa_cases.ca3m_source(rng, f)) for k, f in enumerate(fams)])
    sq = ffindex.FFIndex(prefix + "_sequence.ffdata")
    ca = ffindex.FFIndex(prefix + "_ca3m.ffdata")
    seqs = hhg.capi.SeqDb.make(bytes(sq.data), sq.offsets, sq.lengths)
    for k in range(len(ca.names)):
        hhg.capi.ca3m_parse(bytes(ca.record(k)), seqs)          # raises on a record the reference would exit on
    refs = _reference([_job(prefix, prep=True, name=name) for name in ca.names], tmp_path)
    pb = refshim.pb()
    for k, (name, ref) in enumerate(zip(ca.names, refs)):
        _cmp(hhg.capi.ca3m_to_hmm(gpu_ctx, bytes(ca.record(k)), seqs, pb), ref, f"{name} ({fams[k]})")
    for r in refs:                # compressed records carry no ss rows
        r["ss_pred"] = r["ss_conf"] = np.zeros(r["L"] + 2, np.uint8)
    db = hhg.TargetDB.from_ca3m(gpu_ctx, bytes(ca.data), ca.offsets, ca.lengths, seqs, refshim.R(), pb)
    _check_shard(db, _expected_shard(refs), "compressed database")
    db.close(); sq.close(); ca.close()
