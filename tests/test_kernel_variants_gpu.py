"""Every forward-kernel configuration the library can be switched to must produce the oracle's bits: strip heights
8 / 12 / 16 (HHG_STRIP_ROWS), work-item group sizes (HHG_GROUP_JOBS).  Also a stress run of the tagged-slot strip
hand-off (many epochs, many strips, concurrent contexts)."""
import contextlib
import os
import threading

import numpy as np
import pytest

from tests.test_viterbi_gpu import _check_against_oracle
from tests.util import bits, golden

pytestmark = pytest.mark.gpu


@contextlib.contextmanager
def env_ctx(hhg, **env):
    old = {k: os.environ.get(k) for k in env}
    os.environ.update({k: str(v) for k, v in env.items()})
    try:
        ctx = hhg.Context()
    finally:
        for k, v in old.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v
    try:
        yield ctx
    finally:
        ctx.close()


CONFIGS = [dict(HHG_STRIP_ROWS=16), dict(HHG_STRIP_ROWS=16, HHG_GROUP_JOBS=1), dict(HHG_STRIP_ROWS=16, HHG_GROUP_JOBS=7),
           dict(HHG_STRIP_ROWS=12), dict(HHG_STRIP_ROWS=8), dict(HHG_STRIP_ROWS=8, HHG_GROUP_JOBS=3)]


@pytest.mark.parametrize("cfg", CONFIGS, ids=lambda c: ",".join(f"{k[4:]}={v}" for k, v in c.items()))
def test_all_kernel_configurations_match_oracle(hhg, oracle, cfg):
    from hhsuite_b200 import synth
    G = golden()
    rng = np.random.default_rng(11)
    qp, qtr, qss, qpav, qcols = synth.query_profile(211, 9)     # 14 / 18 / 27 strips, not a multiple of R
    lens = [1, 2, 33, 64, 199, 200, 350, 700] + list(rng.integers(20, 300, 40))
    tg = [synth.prepared_profile(int(L), rng, qcols if k % 3 == 0 else None, noise=0.3) for k, L in enumerate(lens)]
    with env_ctx(hhg, **cfg) as ctx:
        _check_against_oracle(hhg, ctx, oracle, (qp, qtr, qss), tg)
        _check_against_oracle(hhg, ctx, oracle, (qp, qtr, qss), tg, S33=G["S33"], use_ss=True)
        _check_against_oracle(hhg, ctx, oracle, (qp, qtr, qss), tg, local=False, egq=0.3, egt=0.1)
        ids = rng.permutation(len(tg))[:17].astype(np.int32)
        _check_against_oracle(hhg, ctx, oracle, (qp, qtr, qss), tg, ids=ids)


@pytest.mark.parametrize("cfg", [CONFIGS[0], CONFIGS[4]], ids=["R16", "R8"])
def test_long_query_many_strips(hhg, oracle, cfg):
    """Lq=1500: 94 (R=16) / 188 (R=8) strips per job."""
    from hhsuite_b200 import synth
    rng = np.random.default_rng(15)
    qp, qtr, qss, qpav, qcols = synth.query_profile(1500, 7)
    tg = [synth.prepared_profile(L, rng, qcols if k % 2 == 0 else None, noise=0.3)
          for k, L in enumerate([1200, 333, 200, 64, 30])]
    with env_ctx(hhg, **cfg) as ctx:
        _check_against_oracle(hhg, ctx, oracle, (qp, qtr, qss), tg)


def test_handoff_stress_many_epochs_and_concurrent_contexts(hhg, oracle):
    """The strip hand-off relies on tagged 64-bit words (relaxed loads and stores, no fences).  Hammer it: small
    strips (R=8 -> 50 strips), 300 runs of the same plan (slot memory is reused, only the epoch in the tag
    changes), three contexts on their own streams and host threads at once, as hhblits_omp drives the path
    (src/hhblits_omp.cpp:119-138).  Every run must reproduce the first run's bits; the first run is checked
    against the oracle."""
    from hhsuite_b200 import synth
    rng = np.random.default_rng(21)
    qp, qtr, qss, qpav, qcols = synth.query_profile(400, 4)
    tg = [synth.prepared_profile(int(L), rng, qcols if k % 5 == 0 else None, noise=0.3)
          for k, L in enumerate(rng.integers(30, 400, 700))]
    errors = []

    def worker(seed):
        try:
            with env_ctx(hhg, HHG_STRIP_ROWS=8, HHG_GROUP_JOBS=1 + 20 * seed) as ctx:
                ctx.set_query(qp, qtr)
                db = hhg.TargetDB.from_profiles(ctx, tg)
                plan = hhg.Plan(ctx, db)
                plan.run()
                ref, _ = plan.fetch(want_paths=False)
                ref = ref.copy()
                if seed == 0:
                    for k in (0, 1, 350, 699):
                        sc, i2, j2, bt = oracle.viterbi(qp, qtr, tg[k][0], tg[k][1])
                        assert bits(ref[k]["score"]) == bits(sc) and (ref[k]["i2"], ref[k]["j2"]) == (i2, j2)
                for it in range(300):
                    plan.run()
                    if it % 50 == 49:
                        h, _ = plan.fetch(want_paths=False)
                        assert np.array_equal(h.view(np.uint8), ref.view(np.uint8)), (seed, it)
                plan.close(); db.close()
        except BaseException as e:   # noqa: BLE001
            errors.append((seed, repr(e)))

    th = [threading.Thread(target=worker, args=(s,)) for s in range(3)]
    for t in th:
        t.start()
    for t in th:
        t.join()
    assert not errors, errors
