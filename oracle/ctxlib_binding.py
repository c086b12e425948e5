"""ctypes binding of oracle/_ref/libhhref_ctxlib.so (oracle/ctxlib_shim.cpp): the compiled, unmodified reference's
generative context-library engine.  TEST INFRASTRUCTURE: only tests and tools load it.  LibRef() raises
FileNotFoundError when oracle/_ref was not built (oracle/ctxlib_ref.mk needs the reference tree)."""
import ctypes as C
import os

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
c_f32p = C.POINTER(C.c_float)

# cs::Admix classes by name, as RefShim.context_pc_crf takes them
ADMIX_CLASSES = ("constant", "csblast", "hhsearch")


def _f32(a):
    return np.ascontiguousarray(a, np.float32)


class LibRef:
    def __init__(self):
        path = os.path.join(HERE, "_ref", "libhhref_ctxlib.so")
        if not os.path.exists(path):
            raise FileNotFoundError(path)
        self.lib = L = C.CDLL(path)
        L.hhref_lib_text.restype = C.c_void_p
        L.hhref_lib_text.argtypes = [C.POINTER(C.c_longlong)]
        L.hhref_lib_pb.argtypes = [c_f32p]
        L.hhref_lib_set_pb.argtypes = [c_f32p]
        L.hhref_lib_error.restype = C.c_char_p
        L.hhref_lib_text_state.argtypes = [C.c_char_p, C.c_longlong, C.c_int, C.POINTER(C.c_int), C.POINTER(C.c_double),
                                           C.c_void_p, C.c_void_p]
        L.hhref_context_pc_lib.argtypes = [C.c_char_p, C.c_longlong, C.c_double, C.c_double, C.c_char_p, C.c_double,
                                           C.c_double, C.c_double, C.c_int, c_f32p, c_f32p, C.c_float, c_f32p, c_f32p]
        L.hhref_context_pc_dispatch.argtypes = [C.c_char_p, C.c_float, C.c_float, C.c_int, C.c_int, c_f32p, c_f32p,
                                                C.c_float, c_f32p, c_f32p]

    def lib_text(self):
        """The data/context_data.lib bytes embedded in the build (4000 profiles, window 13)."""
        n = C.c_longlong()
        ptr = self.lib.hhref_lib_text(C.byref(n))
        return C.string_at(ptr, n.value)

    def pb(self):
        """The background SetSubstitutionMatrix gives (what CalculateAminoAcidBackground reads)."""
        out = np.zeros(20, np.float32)
        self.lib.hhref_lib_pb(out.ctypes.data_as(c_f32p))
        return out

    def set_pb(self, pb):
        """Replace the background pav is computed with (e.g. by RefShim.pb(), which an HHM read has overwritten)."""
        self.lib.hhref_lib_set_pb(_f32(pb).ctypes.data_as(c_f32p))

    def error(self):
        return self.lib.hhref_lib_error().decode(errors="replace")

    def lib_text_state(self, text, k):
        """Profile k of the library `text` as cs::ContextLibrary's reader + TransformToLog leave it ->
        (n_profiles, log prior, log-probs[wlen, 20], pc[20]).  ValueError when the reader refuses the text."""
        wlen = C.c_int(); prior = C.c_double(); pc = np.zeros(20, np.float64)
        fn = self.lib.hhref_lib_text_state
        n = fn(text, len(text), k, C.byref(wlen), C.byref(prior), None, pc.ctypes.data)
        if n == -1:
            raise ValueError(f"the reference's context library reader refused the text: {self.error()}")
        if n < 0:
            raise IndexError(k)
        probs = np.zeros((wlen.value, 20), np.float64)
        fn(text, len(text), k, C.byref(wlen), C.byref(prior), probs.ctypes.data, pc.ctypes.data)
        return n, prior.value, probs, pc

    def context_pc_lib(self, text, csw, csb, f, neff_m, neff_hmm, admix, pca, pcb=0.0, pcc=1.0):
        """cs::LibraryPseudocounts(lib, csw, csb) + the cs::Admix class named admix (one of ADMIX_CLASSES) +
        HMM::AddContextSpecificPseudocounts + CalculateAminoAcidBackground -> (p[(L+2), 20], pav[20])."""
        if admix not in ADMIX_CLASSES:
            raise ValueError(f"admixture class {admix!r} is not one of {ADMIX_CLASSES}")
        f, neff_m = _f32(f), _f32(neff_m)
        L = f.shape[0] - 2
        p = np.zeros((L + 2, 20), np.float32); pav = np.zeros(20, np.float32)
        r = self.lib.hhref_context_pc_lib(text, len(text), float(csw), float(csb), admix.encode(), float(pca), float(pcb),
                                          float(pcc), L, f.ctypes.data_as(c_f32p), neff_m.ctypes.data_as(c_f32p),
                                          float(neff_hmm), p.ctypes.data_as(c_f32p), pav.ctypes.data_as(c_f32p))
        if r == -1:
            raise ValueError(f"the reference's context library reader refused the text: {self.error()}")
        assert r == L, r
        return p, pav

    def context_pc_dispatch(self, path, csw, csb, engine, f, neff_m, neff_hmm):
        """InitializePseudocountsEngine with par.clusterfile = path (a `.lib` file) and par.csw / par.csb (floats), then
        engine 0 (query HMM, HHsearch admixture) or 1 (prefilter profile, CS-BLAST admixture) -> (p, pav)."""
        f, neff_m = _f32(f), _f32(neff_m)
        L = f.shape[0] - 2
        p = np.zeros((L + 2, 20), np.float32); pav = np.zeros(20, np.float32)
        r = self.lib.hhref_context_pc_dispatch(str(path).encode(), float(csw), float(csb), int(engine), L,
                                               f.ctypes.data_as(c_f32p), neff_m.ctypes.data_as(c_f32p), float(neff_hmm),
                                               p.ctypes.data_as(c_f32p), pav.ctypes.data_as(c_f32p))
        assert r == L, "InitializePseudocountsEngine built no context library engine"
        return p, pav
