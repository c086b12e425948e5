"""Generate tests/golden/ctxlib_v1.npz from the UNMODIFIED compiled reference (oracle/_ref/libhhref_ctxlib.so, built by
oracle/ctxlib_ref.mk, which needs the reference tree):
    python tests/golden/make_ctxlib_golden.py
Every expected value below comes from reference code paths on the inputs of tests/ctxlib_cases.py:
  * cs::ContextLibrary's reader + TransformToLog (hhref_lib_text_state)   -> every profile of every synthetic library,
                                                                             and which texts it refuses or reads
  * SetSubstitutionMatrix's background pb                               -> pb
  * cs::LibraryPseudocounts(lib, csw, csb) + ConstantAdmix / CSBlastAdmix  -> p (one digest per row) and pav
    / HHsearchAdmix + HMM::AddContextSpecificPseudocounts
    + CalculateAminoAcidBackground (hhref_context_pc_lib)
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from oracle.ctxlib_binding import LibRef  # noqa: E402
from tests import ctxlib_cases as cc  # noqa: E402


def main():
    R = LibRef()
    G = {"pb": R.pb()}                     # the background of CalculateAminoAcidBackground, so pav needs no reference
    cases = cc.golden_cases()
    for key, text, (csw, csb), adm, (f, neff_m, neff_hmm) in cases:
        p, pav = R.context_pc_lib(text, csw, csb, f, neff_m, neff_hmm, *cc.admix_args(adm))
        G[f"h/{key}"] = cc.input_digest(text, csw, csb, f, neff_m, neff_hmm, adm)
        G[f"d/{key}"] = cc.row_digests(p)
        G[f"pav/{key}"] = pav
    print("pseudocounts", len(cases))
    for tag, text in cc.libraries():
        n, _, probs0, _ = R.lib_text_state(text, 0)
        digests = np.zeros(n, np.uint64)
        for k in range(n):
            _, prior, probs, pc = R.lib_text_state(text, k)
            digests[k] = cc.state_digest(prior, probs, pc)
        G[f"h/state/{tag}"] = cc.text_digest(text)
        G[f"state/{tag}"] = digests
        G[f"window/{tag}"] = np.int32(probs0.shape[0])
    for tag, text in cc.refused_by_both():
        try:
            R.lib_text_state(text, 0)
            raise AssertionError(f"the reference reads {tag!r}")
        except ValueError:
            G[f"refused/{tag}"] = cc.text_digest(text)
    for tag, text, _ in cc.refused_by_library():
        G[f"h/accepted/{tag}"] = cc.text_digest(text)
        G[f"accepted/{tag}"] = np.int32(R.lib_text_state(text, 0)[0])
    np.savez_compressed(os.path.join(ROOT, "tests", "golden", "ctxlib_v1.npz"), **G)
    print(len(G), "arrays")


if __name__ == "__main__":
    main()
