"""CPU tests of the context-specific (CRF) pseudocounts on the inputs of tests/crf_cases.py: the library's `.crf` parser
against the reference's cs::Crf reader on synthetic libraries and on texts a reader must refuse, and the host tail
(log-sum-exp over the states, admixture, normalisation) under every admixture.  The reference's side of the custom
libraries and admixtures is tests/golden/crf_v1.npz (tests/golden/make_crf_golden.py); the first test ties those goldens
to the live compiled reference.  The context scores the CUDA kernel produces are restated with numpy in its summation
order (tests/test_crf_cpu.py)."""
import numpy as np
import pytest

from tests import crf_cases
from tests.test_crf_cpu import _scores


def _crf(text):
    from hhsuite_b200 import capi
    return capi.Crf(None, text)


@pytest.fixture(scope="module")
def G():
    with crf_cases.golden() as z:
        yield z


def test_goldens_of_the_default_engines_equal_live_reference(refshim, G):
    """The goldens were made by the reference entry that takes the library text and the admixture class; wherever
    that is the embedded context_data.crf with a default admixture, they equal what the engines
    InitializePseudocountsEngine builds compute now, on this host, bit for bit."""
    text = refshim.crf_text()
    cases = crf_cases.golden_cases(text)
    n = 0
    for key, t, adm, (f, neff_m, neff_hmm) in cases["tail"] + cases["admix"]:
        if t != text or tuple(adm) not in (crf_cases.ADMIX_HHM, crf_cases.ADMIX_PREFILTER):
            continue
        p, pav = refshim.context_pc(f, neff_m, neff_hmm, engine=0 if tuple(adm) == crf_cases.ADMIX_HHM else 1)
        crf_cases.compare(p, pav, crf_cases.expected(G, key, t, adm, (f, neff_m, neff_hmm)), key)
        n += 1
    assert n == 2 * (len(crf_cases.tail_profiles()) + len(crf_cases.family("edges")) + 5 + 3)


@pytest.mark.parametrize("tag,text", crf_cases.libraries(), ids=[t for t, _ in crf_cases.libraries()])
def test_parser_equals_reference_reader(G, tag, text):
    """Every state of every synthetic library: emission pseudocounts (UpdatePseudocounts' long-double sum), bias and
    every context weight, '*' included (the reader's INT_MAX / 1000)."""
    assert np.array_equal(G[f"h/state/{tag}"], crf_cases.text_digest(text)), tag
    want = G[f"state/{tag}"]
    crf = _crf(text)
    assert (crf.n_states, crf.window) == (len(want), int(G[f"window/{tag}"]))
    pc = crf.pc()
    got = np.array([crf_cases.state_digest(pc[k], *crf.state(k)[::-1]) for k in range(crf.n_states)], np.uint64)
    bad = np.flatnonzero(got != want)
    assert len(bad) == 0, (tag, "states differ from the reference reader's, the first is", int(bad[0]))
    if b"*" in text:
        assert any((crf.state(k)[0] == 2147483647 / 1000).any() for k in range(crf.n_states))
    crf.close()


@pytest.mark.parametrize("tag,text", crf_cases.refused_by_both(), ids=[t for t, _ in crf_cases.refused_by_both()])
def test_parser_refuses_what_reference_refuses(G, tag, text):
    from hhsuite_b200 import capi
    assert np.array_equal(G[f"refused/{tag}"], crf_cases.text_digest(text)), tag
    with pytest.raises(capi.HhgError):
        _crf(text)


def test_parser_limits():
    """What only the library refuses, each with a message naming the problem: windows longer than 63 columns (the
    kernel's shared-memory window), even windows (the reference's reader asserts on them), a state without a PC row
    (the reference would read uninitialised weights) and a state whose window differs from the library's."""
    from hhsuite_b200 import capi
    texts = {tag: text for tag, text, _ in crf_cases.refused_by_library()}
    texts["window 4"] = crf_cases.even_window()
    messages = {"window 65": "window length 65 .*odd and 1..63", "window 4": "window length 4 .*odd and 1..63",
                "a state without a PC row": "without a PC row",
                "a state LENG differing from the CRF's": "window length differs"}
    assert set(texts) == set(messages)
    for tag, text in texts.items():
        with pytest.raises(capi.HhgError, match=messages[tag]):
            _crf(text)


def test_reference_reads_what_only_the_library_refuses(G):
    """The other side of test_parser_limits: the reference's reader takes these texts, so the limits are the
    library's own, not a reader parity gap.  None of them is used for pseudocounts."""
    for tag, text, reason in crf_cases.refused_by_library():
        assert np.array_equal(G[f"h/accepted/{tag}"], crf_cases.text_digest(text)), tag
        assert int(G[f"accepted/{tag}"]) >= 1, tag


@pytest.mark.parametrize("ai", range(len(crf_cases.ADMIXTURES)), ids=[str(a) for a in crf_cases.ADMIXTURES])
def test_tail_equals_reference_for_every_admixture(refshim, G, ai):
    """hhg_crf_tail_host on numpy context scores: the embedded library on clipped windows, single sequences, a diverse
    and a conserved profile, and one synthetic library with '*' weights, under each admixture of the table."""
    from hhsuite_b200 import capi
    adm = crf_cases.ADMIXTURES[ai]
    crfs = {}
    for key, text, a, prof in crf_cases.golden_cases(refshim.crf_text())["tail"]:
        if not key.startswith(f"tail/{ai}/"):
            continue
        crf = crfs.setdefault(text, _crf(text))
        f, neff_m, neff_hmm = prof
        L = f.shape[0] - 2
        got = crf.tail_host(_scores(crf, f, neff_m), f, neff_m, capi.Admix(*adm))
        crf_cases.compare(got, None, crf_cases.expected(G, key, text, a, prof), key, rows=slice(1, L + 1))
    assert len(crfs) == 2
    for crf in crfs.values():
        crf.close()
