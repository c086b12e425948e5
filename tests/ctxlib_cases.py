"""Seeded inputs of the context-library pseudocount tests (the generative engine `-contxt <file>` selects for any file
that is not a `.crf`), shared by the CPU and GPU tests: synthetic libraries written the way cs::ContextLibrary::Write
and ContextProfile::Write write them, texts a reader must refuse, the window weights (-csw / -csb) to run them with and
the table of golden cases.  The count profiles and the admixtures are those of tests/crf_cases.py."""
import os

import numpy as np

from tests import crf_cases
from tests.crf_cases import ADMIX_HHM, ADMIX_PREFILTER, ADMIXTURES, admix_args, row_digests, text_digest  # noqa: F401

AA = crf_cases.AA
F32 = lambda x: float(np.float32(x))   # noqa: E731  hhblits keeps par.csw / par.csb as floats

CSW, CSB = F32(1.6), F32(0.85)        # -csw / -csb defaults as the engine receives them
# (csw, csb): the defaults, no context weight at all, a window of the centre column only, no decay
WEIGHTS = [(CSW, CSB), (0.0, CSB), (2.5, 0.0), (CSW, 1.0)]


# --------------------------------------------------------------------------------------------- synthetic context libraries
def lib_text(profiles, W, is_log, names=None, color=True):
    """A context library as cs::ContextLibrary::Write + ContextProfile::Write write it (src/cs/context_library-inl.h:71-78,
    context_profile-inl.h:147-176).  profiles: [(prior, rows[W][20] of ints or "*")]; names[k] or None (no NAME line);
    color False leaves out the COLOR lines, which the reader skips when they are missing."""
    out = ["ContextLibrary\n", f"SIZE\t{len(profiles)}\n", f"LENG\t{W}\n"]
    for k, (prior, rows) in enumerate(profiles):
        out.append("ContextProfile\n")
        if names is not None and names[k]:
            out.append(f"NAME\t{names[k]}\n")
        out.append("PRIOR\t%-10.8g\n" % prior)
        if color:
            out.append("COLOR\t1.00,0.36,1.00\n")
        out.append(f"ISLOG\t{'T' if is_log else 'F'}\nLENG\t{len(rows)}\nALPH\t20\n")
        out.append("PROBS" + "".join("\t" + a for a in AA) + "\n")
        for i, row in enumerate(rows):
            out.append(str(i + 1) + "".join("\t" + str(v) for v in row) + "\n")
        out.append("//\n")
    return "".join(out).encode()


def random_profiles(rng, K, W):
    """K profiles of window W: priors across many decades, values (-1000 * log2 p) mostly 0..15000 with a few negative
    ones (p > 1) and a few up to 2^-1060, still a normal double."""
    profiles = []
    for _ in range(K):
        rows = rng.integers(0, 15001, (W, 20))
        rare = rng.random((W, 20))
        rows[rare < 0.01] = rng.integers(-3000, 0, int((rare < 0.01).sum()))
        rows[rare > 0.995] = rng.integers(15000, 1060001, int((rare > 0.995).sum()))
        profiles.append((float(10.0 ** rng.uniform(-8, -0.5)), rows.tolist()))
    return profiles


# (K, W, ISLOG, NAME lines, COLOR lines): K around the score kernel's block of 256 threads, W up to the 63 columns it holds
LIBRARIES = [(1, 1, False, False, True), (2, 3, True, True, False), (255, 13, False, True, True),
             (256, 15, True, False, True), (257, 63, False, True, False), (1000, 13, True, True, True),
             (1, 63, True, False, False), (256, 1, False, True, True), (1000, 3, False, False, True)]


def library(K, W, is_log=False, names=False, color=True, seed=0):
    rng = np.random.default_rng([seed, K, W, int(is_log), int(names), int(color), 11])
    nm = [f"P{k}" if rng.random() < 0.7 else "" for k in range(K)] if names else None
    return lib_text(random_profiles(rng, K, W), W, is_log, nm, color)


def _tag(K, W, is_log, names, color):
    return f"K={K} W={W} ISLOG {'T' if is_log else 'F'}{' names' if names else ''}{' color' if color else ''}"


def libraries():
    """[(tag, text)] of every synthetic library."""
    return [(_tag(*spec), library(*spec)) for spec in LIBRARIES]


def window(text):
    return int(text.split(b"\n")[2].split(b"\t")[1])


def _edit(text, old, new, count=1):
    assert old in text
    return text.replace(old, new, count)


def refused_by_both():
    """[(tag, text)]: texts the reference's reader and the library's both refuse."""
    base = library(3, 5, names=True, seed=7)
    rows = base.split(b"\n")
    return [
        # the trailing line keeps the reader off end-of-file, where it would test a buffer fgets did not fill
        ("SIZE larger than the profiles given", _edit(base, b"SIZE\t3", b"SIZE\t4") + b"END\n"),
        ("a profile with fewer rows than LENG", b"\n".join(r for r in rows if not r.startswith(b"5\t"))),
        ("not a context library", b"ContextLibrarx\n" + base[len(b"ContextLibrary\n"):]),
        ("a CRF", crf_cases.library(2, 3)),
        ("a profile without PRIOR", _edit(base, b"PRIOR", b"PRIAR")),
        ("alphabet size 21", _edit(base, b"ALPH\t20", b"ALPH\t21")),
    ]


def refused_by_library():
    """[(tag, text, message)]: texts only the library refuses, each a deliberate limit or a text whose result would be
    NaN; message is what the refusal says.  Even windows are not given to the reference: its reader asserts on them."""
    base = library(3, 5, seed=8)
    first_row = base.index(b"\n1\t") + 1
    star = base[:first_row] + b"1\t*" + base[base.index(b"\t", first_row + 2):]
    under = base[:first_row] + b"1\t1075000" + base[base.index(b"\t", first_row + 2):]
    second = base.index(b"ContextProfile", base.index(b"ContextProfile") + 1)
    third = base.index(b"ContextProfile", second + 1)
    other = lib_text(random_profiles(np.random.default_rng(9), 1, 7), 7, False)
    other_len = base[:second] + other[other.index(b"ContextProfile"):] + base[third:]
    twice = base[:base.index(b"\n3\t") + 1] + b"2" + base[base.index(b"\n3\t") + 2:]
    return [
        ("window 65", library(2, 65, seed=1), "window length 65 .*odd and 1..63"),
        ("a '*' value", star, r"profile 0, column 1, amino acid 0: 2\^\(-2147483647/1000\) is not a positive finite"),
        ("a value whose probability underflows", under, r"profile 0, column 1, amino acid 0: 2\^\(-1075000/1000\)"),
        ("a profile LENG differing from the library's", other_len, "profile 1 has window length 7, the library 5"),
        ("a row given twice", twice, "profile 0, column 2 is given twice"),
        ("a negative PRIOR", _edit(base, b"PRIOR\t", b"PRIOR\t-"), "PRIOR of profile 0 is not a probability"),
    ]


def even_window():
    return library(2, 4, seed=2)


def empty_library():
    """SIZE 0: the reference reads an empty library (and every column's pseudocounts would be 0 / 0)."""
    return b"ContextLibrary\nSIZE\t0\nLENG\t13\n"


# --------------------------------------------------------------------------------------------------------------- goldens
# The synthetic libraries under every admixture and every window weight pair read tests/golden/ctxlib_v1.npz: what the
# reference's cs::LibraryPseudocounts computed on these inputs (tests/golden/make_ctxlib_golden.py), so they need no
# compiled reference.  Keys and digests follow tests/golden/crf_v1.npz (tests/crf_cases.py).
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ctxlib_v1.npz")


def golden():
    return np.load(GOLDEN)


def input_digest(text, csw, csb, f, neff_m, neff_hmm, adm):
    return crf_cases.input_digest(text, f, neff_m, neff_hmm, tuple(adm) + (csw, csb))


def state_digest(prior, probs, pc):
    """Digest of one profile as the reader leaves it: log prior, log-probabilities and central column, float64 bits."""
    return crf_cases.state_digest(pc, prior, probs)


def profiles_for(W):
    """Count profiles of a library of window W: the edge family relative to W and a 200-column diverse profile."""
    return crf_cases.family("edges", W=W) + [("diverse L=200", crf_cases.diverse(np.random.default_rng(200), 200))]


def golden_cases():
    """[(key, text, (csw, csb), adm, (f, neff_m, neff_hmm))]: every synthetic library under every admixture and every
    weight pair, the count profile rotating through profiles_for(W)."""
    out = []
    for tag, text in libraries():
        profs = profiles_for(window(text))
        for ai, adm in enumerate(ADMIXTURES):
            for wi, wts in enumerate(WEIGHTS):
                ptag, prof = profs[(ai * len(WEIGHTS) + wi) % len(profs)]
                out.append((f"lib/{tag}/{ai}/{wi}/{ptag}", text, wts, adm, prof))
    return out


def expected(G, key, text, wts, adm, prof):
    """(row digests, pav) the reference computed for this case, after checking the golden holds these very inputs."""
    f, neff_m, neff_hmm = prof
    assert f"h/{key}" in G.files, f"no golden for {key}"
    assert np.array_equal(G[f"h/{key}"], input_digest(text, *wts, f, neff_m, neff_hmm, adm)), \
        f"the inputs of {key} are not those tests/golden/ctxlib_v1.npz was made from"
    return G[f"d/{key}"], G[f"pav/{key}"]


compare = crf_cases.compare
