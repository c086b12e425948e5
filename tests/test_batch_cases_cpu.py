"""The query-batch builders of tests/batch_cases.py (no GPU): the numpy null model is the reference's bit for bit,
every length family is present, and the restated plan rules give the strip heights and waves the GPU tests expect."""
import numpy as np
import pytest

from tests import batch_cases as bc
from tests.util import bits, golden


@pytest.mark.parametrize("columnscore", [0, 1, 2, 3])
@pytest.mark.parametrize("name", ["t150", "tself"])
def test_numpy_null_model_matches_reference_goldens(name, columnscore):
    """nm_<name>_p_cs<k> of golden_v1.npz are HMM::IncludeNullModelInHMM of the compiled reference."""
    G = golden()
    got = bc.null_model(G[f"nm_{name}_praw"], G[f"nm_{name}_pav"], G["q_pav"], G["pb"], columnscore)
    assert np.array_equal(bits(got), bits(G[f"nm_{name}_p_cs{columnscore}"]))


@pytest.mark.parametrize("kind", ["scan", "survivors"])
def test_builders_hit_every_length_family(kind):
    b = bc.make_batch(kind)
    lq, lt = bc.request_lengths(b)
    assert set(bc.QUERY_LENGTHS) <= set(b["q_lens"].tolist())
    assert set(bc.TARGET_EDGES) <= set(lt.tolist())
    assert lt.max() == 3000
    cnt = np.bincount(b["req_q"], minlength=len(b["q_lens"]))
    assert set(bc.COUNT_EDGES) <= set(cnt.tolist())
    assert cnt.max() > (380 if kind == "scan" else 33)
    pairs = b["req_q"].astype(np.int64) * 100000 + b["ids"]
    assert len(np.unique(pairs)) < len(pairs)                          # duplicate (query, target) requests
    assert np.any(np.diff(b["req_q"]) < 0)                             # queries interleaved, not grouped
    assert bc.make_batch(kind)["ids"].tobytes() == b["ids"].tobytes()  # seeded


@pytest.mark.parametrize("kind,R", [("scan", 16), ("survivors", 8)])
def test_restated_strip_height_rule(kind, R):
    b = bc.make_batch(kind)
    assert bc.strip_rows(b["q_lens"], b["req_q"], bc.H100_SMS) == R
    assert bc.strip_rows(b["q_lens"], b["req_q"], bc.H100_SMS, forced=12) == 12
    n16 = bc.items16(b["q_lens"], b["req_q"])
    assert (n16 >= 4 * bc.H100_SMS * 8) == (R == 16)


def test_restated_jobs_and_waves():
    """Job geometry and the memory waves of the scan batch at the wave test's budget: at least five waves, one job
    larger than the budget, and a wave boundary inside one query's jobs."""
    b = bc.make_batch("scan")
    lq, lt = bc.request_lengths(b)
    jobs = bc.plan_jobs(b["q_lens"], b["req_q"], lt, 16)
    cnt = np.bincount(b["req_q"], minlength=len(b["q_lens"]))
    assert len(jobs) == sum((int(c) + 31) // 32 for c in cnt)
    assert bc.padded_cells(jobs, 16) >= float((lq.astype(np.int64) * lt).sum())
    budget = bc.bt_budget(bc.SCAN_WAVE_GB)
    sizes = bc.wave_sizes(jobs, 16, budget)
    assert len(sizes) >= 5 and sum(sizes) == len(jobs)
    assert max(bc.job_bt_bytes(j, 16) for j in jobs) > budget
    bounds = np.cumsum(sizes)[:-1]
    q_of_job = [j[0] for j in jobs]
    assert any(q_of_job[e - 1] == q_of_job[e] for e in bounds)



def test_plan_too_large_request_count():
    """65 600 requests of Lq = 32 767 against 1-column targets pass 2^31 - 1 path bytes."""
    assert 65600 * (bc.MAX_LEN + 1 + 2) > bc.PATH_LIMIT
