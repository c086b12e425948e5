"""CPU tests of the context-library pseudocounts (hhg_context_library_*: the generative engine `-contxt <file>` picks
for a file that is not a `.crf`): the library's reader against cs::ContextLibrary's reader + TransformToLog, profile by
profile and bit for bit, on the reference's context_data.lib and on the synthetic libraries of tests/ctxlib_cases.py;
every refusal; the score kernel run by the CPU emulation (tests/emul/ctxlib_emul.cpp) plus the host tail against the
reference's cs::LibraryPseudocounts under every admixture and every window weight pair; the goldens against the live
reference; and the reference's own engine dispatch against the direct construction the other tests use."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from tests import crf_cases
from tests import ctxlib_cases as cc
from tests.util import ROOT, bits


@pytest.fixture(scope="module")
def emul(tmp_path_factory):
    """k_lib_scores on the CPU emulation, compiled into a temporary directory."""
    lib = str(tmp_path_factory.mktemp("emul") / "libctxlibemul.so")
    subprocess.check_call(["g++", "-O1", "-std=c++20", "-ffp-contract=off", "-fPIC", "-shared", "-pthread", "-DHHG_EMUL",
                           "-o", lib, os.path.join(ROOT, "tests", "emul", "ctxlib_emul.cpp")])
    L = C.CDLL(lib)
    L.emul_lib_scores.argtypes = [C.c_int, C.c_int, C.c_int] + [C.c_void_p] * 5
    return L


@pytest.fixture(scope="module")
def libref():
    from oracle.ctxlib_binding import LibRef
    try:
        return LibRef()
    except (FileNotFoundError, OSError) as e:
        pytest.skip(f"compiled reference not available: {e}")


@pytest.fixture(scope="module")
def G():
    with cc.golden() as z:
        yield z


def _lib(text, wts=(cc.CSW, cc.CSB)):
    from hhsuite_b200 import capi
    return capi.ContextLibrary(None, text, *wts)


def _states(lib):
    pc = lib.pc()
    return np.array([cc.state_digest(lib.state(k)[1], lib.state(k)[0], pc[k]) for k in range(lib.n_states)], np.uint64)


def test_reader_equals_reference_on_context_data_lib(libref):
    """All 4000 profiles of the shipped library: log prior, 13 x 20 log-probabilities and the linear central column."""
    text = libref.lib_text()
    lib = _lib(text)
    assert (lib.n_states, lib.window) == (4000, 13)
    want = np.array([cc.state_digest(*libref.lib_text_state(text, k)[1:]) for k in range(4000)], np.uint64)
    bad = np.flatnonzero(_states(lib) != want)
    assert len(bad) == 0, ("profiles differ from the reference reader's, the first is", int(bad[0]))
    lib.close()


@pytest.mark.parametrize("tag,text", cc.libraries(), ids=[t for t, _ in cc.libraries()])
def test_reader_equals_reference_reader(G, tag, text):
    """Every profile of every synthetic library (ISLOG T and F, with and without NAME and COLOR lines)."""
    assert np.array_equal(G[f"h/state/{tag}"], cc.text_digest(text)), tag
    want = G[f"state/{tag}"]
    lib = _lib(text)
    assert (lib.n_states, lib.window) == (len(want), int(G[f"window/{tag}"]))
    bad = np.flatnonzero(_states(lib) != want)
    assert len(bad) == 0, (tag, "profiles differ from the reference reader's, the first is", int(bad[0]))
    lib.close()


@pytest.mark.parametrize("tag,text", cc.refused_by_both(), ids=[t for t, _ in cc.refused_by_both()])
def test_reader_refuses_what_reference_refuses(G, tag, text):
    from hhsuite_b200 import capi
    assert np.array_equal(G[f"refused/{tag}"], cc.text_digest(text)), tag
    with pytest.raises(capi.HhgError):
        _lib(text)


def test_reader_limits():
    """What only the library refuses, each with a message naming the profile and column: windows over 63 columns or
    even, SIZE < 1, a profile LENG other than the library's, a row given twice, a negative PRIOR, '*' and any value
    whose probability is 0 in double, and window weights that are not finite."""
    from hhsuite_b200 import capi
    cases = [(tag, text, msg) for tag, text, msg in cc.refused_by_library()]
    cases += [("window 4", cc.even_window(), "window length 4 .*odd and 1..63"),
              ("SIZE 0", cc.empty_library(), "SIZE 0 is not a positive number of profiles")]
    for tag, text, msg in cases:
        with pytest.raises(capi.HhgError, match=msg):
            _lib(text)
    good = cc.library(2, 3)
    for wts in ((float("nan"), cc.CSB), (cc.CSW, float("inf"))):
        with pytest.raises(capi.HhgError, match="not finite"):
            _lib(good, wts)


def test_reference_reads_what_only_the_library_refuses(G):
    """The other side of test_reader_limits: the reference's reader takes these texts, so the limits are the library's
    own, not a reader parity gap."""
    for tag, text, _ in cc.refused_by_library():
        assert np.array_equal(G[f"h/accepted/{tag}"], cc.text_digest(text)), tag
        assert int(G[f"accepted/{tag}"]) >= 1, tag


def test_each_engine_refuses_the_others_text():
    """hhg_crf_create keeps refusing anything but a CRF; the library reader refuses a CRF."""
    from hhsuite_b200 import capi
    with pytest.raises(capi.HhgError, match="class id 'CRF'"):
        capi.Crf(None, cc.library(2, 3))
    with pytest.raises(capi.HhgError, match="class id 'ContextLibrary'"):
        _lib(crf_cases.library(2, 3))


def _emul_scores(emul, lib, f, neff_m):
    """k_lib_scores on the CPU emulation with the library's own weights and window weights."""
    L = f.shape[0] - 2
    K, W = lib.n_states, lib.window
    c = (W - 1) // 2
    w = np.zeros((W, 20, K)); bias = np.zeros(K)
    for k in range(K):
        w[:, :, k], bias[k] = lib.state(k)
    ww = np.zeros(W)
    ww[c] = lib.weight_center
    for d in range(1, c + 1):
        ww[c - d] = ww[c + d] = lib.weight_center * lib.weight_decay ** d      # C pow, as cs::Emission
    counts = np.ascontiguousarray((f[1:L + 1] * neff_m[1:L + 1, None]).astype(np.float32).astype(np.float64))
    score = np.zeros((L, K))
    emul.emul_lib_scores(L, K, W, w.ctypes.data, bias.ctypes.data, ww.ctypes.data, counts.ctypes.data, score.ctypes.data)
    return score


@pytest.mark.parametrize("ai", range(len(cc.ADMIXTURES)), ids=[str(a) for a in cc.ADMIXTURES])
def test_emulated_kernel_and_tail_equal_reference(libref, emul, ai):
    """The score kernel (emulated) + hhg_crf_tail_host against hhref_context_pc_lib under one admixture and every
    window weight pair, on a 257-profile library of window 13 and short profiles clipped by the window."""
    from hhsuite_b200 import capi
    adm = cc.ADMIXTURES[ai]
    text = cc.library(257, 13, False, True, True)
    profiles = crf_cases.family("edges")[:8]
    for wi, wts in enumerate(cc.WEIGHTS):
        lib = _lib(text, wts)
        tag, (f, neff_m, neff_hmm) = profiles[(ai + wi) % len(profiles)]
        L = f.shape[0] - 2
        got = lib.tail_host(_emul_scores(emul, lib, f, neff_m), f, neff_m, capi.Admix(*adm))
        want, _ = libref.context_pc_lib(text, *wts, f, neff_m, neff_hmm, *cc.admix_args(adm))
        assert np.array_equal(bits(got[1:L + 1]), bits(want[1:L + 1])), (tag, wts)
        lib.close()


def test_emulated_kernel_on_context_data_lib(libref, emul):
    """The shipped library with both hhblits engines on a clipped profile."""
    from hhsuite_b200 import capi
    text = libref.lib_text()
    lib = _lib(text)
    f, neff_m, neff_hmm = crf_cases.family("diverse")[0][1]
    L = f.shape[0] - 2
    score = _emul_scores(emul, lib, f, neff_m)
    for adm in (cc.ADMIX_HHM, cc.ADMIX_PREFILTER):
        got = lib.tail_host(score, f, neff_m, capi.Admix(*adm))
        want, _ = libref.context_pc_lib(text, cc.CSW, cc.CSB, f, neff_m, neff_hmm, *cc.admix_args(adm))
        assert np.array_equal(bits(got[1:L + 1]), bits(want[1:L + 1])), adm
    lib.close()


def test_goldens_equal_live_reference(libref, G):
    """Every golden case recomputed by the reference on this host, bit for bit."""
    assert np.array_equal(bits(G["pb"]), bits(libref.pb()))
    cases = cc.golden_cases()
    assert len(cases) == len(cc.LIBRARIES) * len(cc.ADMIXTURES) * len(cc.WEIGHTS)
    for key, text, wts, adm, prof in cases:
        p, pav = libref.context_pc_lib(text, *wts, *prof, *cc.admix_args(adm))
        cc.compare(p, pav, cc.expected(G, key, text, wts, adm, prof), key)


def test_reference_dispatch_equals_direct_construction(libref, tmp_path):
    """InitializePseudocountsEngine given a `.lib` file builds the engines the other tests construct directly: the
    library through cs::ContextLibrary + TransformToLog, LibraryPseudocounts(lib, par.csw, par.csb), HHsearch 0.9 / 4.0
    / 1.0 for the query HMM and CS-BLAST 0.8 / 2.0 for the prefilter profile."""
    text = libref.lib_text()
    path = tmp_path / "context_data.lib"
    path.write_bytes(text)
    for (csw, csb) in ((cc.CSW, cc.CSB), (cc.F32(2.5), cc.F32(0.5))):
        for tag, (f, neff_m, neff_hmm) in crf_cases.family("edges")[::4] + crf_cases.family("diverse")[:1]:
            for engine, adm in ((0, cc.ADMIX_HHM), (1, cc.ADMIX_PREFILTER)):
                p, pav = libref.context_pc_dispatch(path, csw, csb, engine, f, neff_m, neff_hmm)
                rp, rpav = libref.context_pc_lib(text, csw, csb, f, neff_m, neff_hmm, *cc.admix_args(adm))
                assert p.tobytes() == rp.tobytes() and pav.tobytes() == rpav.tobytes(), (tag, engine, csw, csb)
