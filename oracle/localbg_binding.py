"""ctypes binding of oracle/_ref/libhhref_localbg.so (oracle/localbg_shim.cpp): the compiled, unmodified reference's
local amino-acid composition correction (-sc 5 / -scwin D).  TEST INFRASTRUCTURE: only tests and tools load it.
LocalBgRef() raises FileNotFoundError when oracle/_ref was not built (oracle/localbg_ref.mk needs the reference
tree)."""
import ctypes as C
import os

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
c_f32p = C.POINTER(C.c_float)


def _p(a):
    return a.ctypes.data_as(c_f32p)


class LocalBgRef:
    MAXL = 4000      # profile capacity of the file readers (the library's HMMs hold 4096 rows)

    def __init__(self):
        path = os.path.join(HERE, "_ref", "libhhref_localbg.so")
        if not os.path.exists(path):
            raise FileNotFoundError(path)
        self.lib = L = C.CDLL(path)
        L.hhlb_local_bg.argtypes = [C.c_int, c_f32p, c_f32p, C.c_int, c_f32p]
        L.hhlb_prepare_query_hhm.argtypes = [C.c_char_p, C.c_int, C.c_int, C.c_int, c_f32p, c_f32p]
        L.hhlb_prepare_template_hhm.argtypes = [C.c_char_p, C.c_int, c_f32p, c_f32p, c_f32p]
        L.hhlb_get_R.argtypes = [c_f32p]

    def local_bg(self, p, pb, D):
        """HMM::DivideBySqrtOfLocalBackgroundFreqs(D, pb) on a copy of p[(L+2), 20]; rows 0 and L+1 stay as they are."""
        p = np.ascontiguousarray(p, np.float32)
        pb = np.ascontiguousarray(pb, np.float32)
        out = np.zeros_like(p)
        if self.lib.hhlb_local_bg(p.shape[0] - 2, _p(p), _p(pb), int(D), _p(out)) < 0:
            raise ValueError(f"hhlb_local_bg: length {p.shape[0] - 2} outside [1, 32767]")
        return out

    def prepare_query_hhm(self, path, columnscore=1, D=40):
        """HMM::Read + PrepareQueryHMM (nocontxt) under -sc columnscore / -scwin D -> (HMM::p [(L+2), 20], pb the reader
        set).  The query stays loaded for prepare_template_hhm."""
        p = np.zeros((self.MAXL + 2, 20), np.float32)
        pb = np.zeros(20, np.float32)
        L = self.lib.hhlb_prepare_query_hhm(str(path).encode(), columnscore, int(D), self.MAXL, _p(p), _p(pb))
        if L < 0:
            raise IOError(f"hhlb_prepare_query_hhm({path}): {L}")
        return p[:L + 2].copy(), pb

    def prepare_template_hhm(self, path):
        """HMM::Read + the steps of PrepareTemplateHMM with the column score and window of the last prepared query
        -> dict(p_raw before IncludeNullModelInHMM, p after it, pb the reader set)."""
        p_raw = np.zeros((self.MAXL + 2, 20), np.float32)
        p = np.zeros_like(p_raw)
        pb = np.zeros(20, np.float32)
        L = self.lib.hhlb_prepare_template_hhm(str(path).encode(), self.MAXL, _p(p_raw), _p(p), _p(pb))
        if L < 0:
            raise IOError(f"hhlb_prepare_template_hhm({path}): {L}")
        return dict(L=L, p_raw=p_raw[:L + 2].copy(), p=p[:L + 2].copy(), pb=pb)

    def R(self):
        out = np.zeros(400, np.float32)
        self.lib.hhlb_get_R(_p(out))
        return out.reshape(20, 20)
