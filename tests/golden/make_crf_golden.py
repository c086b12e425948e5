"""Generate tests/golden/crf_v1.npz from the UNMODIFIED compiled reference (oracle/_ref built from this revision's
oracle/ref_shim.cpp, which needs /root/reference):
    python tests/golden/make_crf_golden.py
Every expected value below comes from reference code paths on the inputs of tests/crf_cases.py:
  * cs::Crf's reader (hhref_crf_text_state)                           -> every state of every synthetic library,
                                                                           and which texts it refuses
  * cs::CrfPseudocounts + ConstantAdmix / CSBlastAdmix / HHsearchAdmix  -> p (one digest per row) and pav
    + HMM::AddContextSpecificPseudocounts + CalculateAminoAcidBackground   (hhref_context_pc_crf)
Before writing, the explicit entry is checked against the engines InitializePseudocountsEngine builds (the two default
admixtures on the embedded context_data.crf), bit for bit.
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from oracle.binding import RefShim  # noqa: E402
from tests import crf_cases as cc  # noqa: E402


def main():
    R = RefShim(nocontxt=True, maxres=4096)
    embedded = R.crf_text()
    G = {}
    for group, cases in cc.golden_cases(embedded).items():
        for key, text, adm, (f, neff_m, neff_hmm) in cases:
            p, pav = R.context_pc_crf(text, f, neff_m, neff_hmm, *cc.admix_args(adm))
            if text == embedded and tuple(adm) in (cc.ADMIX_HHM, cc.ADMIX_PREFILTER):
                want = R.context_pc(f, neff_m, neff_hmm, engine=0 if tuple(adm) == cc.ADMIX_HHM else 1)
                assert p.tobytes() == want[0].tobytes() and pav.tobytes() == want[1].tobytes(), key
            G[f"h/{key}"] = cc.input_digest(text, f, neff_m, neff_hmm, adm)
            G[f"d/{key}"] = cc.row_digests(p)
            G[f"pav/{key}"] = pav
        print(group, len(cases))
    for tag, text in cc.libraries():
        n, _, _, w0 = R.crf_text_state(text, 0)
        digests = np.zeros(n, np.uint64)
        for k in range(n):
            _, pc, bias, w = R.crf_text_state(text, k)
            digests[k] = cc.state_digest(pc, bias, w)
        G[f"h/state/{tag}"] = cc.text_digest(text)
        G[f"state/{tag}"] = digests
        G[f"window/{tag}"] = np.int32(w0.shape[0])
    for tag, text in cc.refused_by_both():
        try:
            R.crf_text_state(text, 0)
            raise AssertionError(f"the reference reads {tag!r}")
        except ValueError:
            G[f"refused/{tag}"] = cc.text_digest(text)
    for tag, text, _ in cc.refused_by_library():
        G[f"h/accepted/{tag}"] = cc.text_digest(text)
        G[f"accepted/{tag}"] = np.int32(R.crf_text_state(text, 0)[0])
    np.savez_compressed(os.path.join(ROOT, "tests", "golden", "crf_v1.npz"), **G)
    print(len(G), "arrays")


if __name__ == "__main__":
    main()
