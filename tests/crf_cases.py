"""Seeded inputs of the context-specific (CRF) pseudocount tests, shared by the CPU and GPU tests: count profiles
(f, Neff_M, Neff_HMM) in shape families, synthetic context libraries written the way cs::Crf::Write writes them, texts
a reader must refuse, and a table of pseudocount admixtures.

A count profile is what HMM::AddContextSpecificPseudocounts reads: f[(L+2)*20] (rows 1..L used), Neff_M[L+1] (entries
1..L used) and the HMM's Neff, which only CalculateAminoAcidBackground uses."""
import hashlib
import os

import numpy as np

AA = "ARNDCQEGHILKMFPSTWYV"          # cs::AA::kIntToChar, the WEIGHTS line of a serialized state
W_DEFAULT = 13                       # window of the embedded context_data.crf
MAX_QUERY = 32767                    # longest query hhg_query_set takes

# (kind, pca, pcb, pcc): hhg_admix of the library.  kind 0 constant (cs::ConstantAdmix), 1 CS-BLAST (cs::CSBlastAdmix),
# 2 HHsearch (cs::HHsearchAdmix); ADMIX_CLASS names the reference's class of each kind.
ADMIX_CLASS = {0: "constant", 1: "csblast", 2: "hhsearch"}
ADMIX_HHM = (2, 0.9, 4.0, 1.0)       # -pc_hhm_contxt_* defaults (query HMM)
ADMIX_PREFILTER = (1, 0.8, 2.0, 1.0)  # -pc_prefilter_contxt_* defaults (prefilter profile)
ADMIXTURES = [
    ADMIX_HHM,
    ADMIX_PREFILTER,
    (0, 1.0, 0.0, 1.0),              # pure context pseudocounts
    (0, 0.5, 0.0, 1.0),
    (0, 0.0, 0.0, 1.0),              # tau = 0: p = counts / Neff
    (1, 0.001, 2.0, 1.0),            # the floor hhblits clamps pc_prefilter_contxt_a to
    (1, 2.0, 2.0, 1.0),              # MIN(1.0, .) takes over for Neff < 4
    (2, 0.9, 4.0, 0.7),              # pcc != 1: the pow branch
    (2, 1.0, 1.5, 2.0),
    (2, 1.5, 4.0, 1.0),              # MIN(1.0, .) takes over for Neff < 2
]


def admix_args(adm):
    """(class name, pca, pcb, pcc) for RefShim.context_pc_crf."""
    kind, a, b, c = adm
    return (ADMIX_CLASS[kind], a, b, c)


# ------------------------------------------------------------------------------------------------------ count profiles
def edge_lengths(W=W_DEFAULT):
    """Query lengths around the window: clipped on both sides (L < W), L = W, and the first and last columns whose
    window lies fully inside (L = W + c and 2W - 1 .. 2W + 1 for c = (W - 1) / 2).  W = 13: 1 2 3 6 7 12 13 14 19 25 26 27."""
    c = (W - 1) // 2
    return sorted({L for L in (1, 2, 3, c, c + 1, W - 1, W, W + 1, W + c, 2 * W - 1, 2 * W, 2 * W + 1) if L >= 1})


def _profile(f_rows, neff_rows, neff_hmm):
    """Wrap rows 1..L in the (L+2)-row f / (L+1)-entry Neff_M layout; the unused rows get plausible values."""
    L = len(f_rows)
    f = np.zeros((L + 2, 20), np.float32)
    f[1:L + 1] = f_rows
    f[0] = f[L + 1] = np.float32(0.05)
    neff_m = np.zeros(L + 1, np.float32)
    neff_m[0] = np.float32(1.0)
    neff_m[1:] = neff_rows
    return f, neff_m, float(np.float32(neff_hmm))


def _dirichlet(rng, L, alpha):
    return rng.dirichlet(np.full(20, alpha), L).astype(np.float32)


def _one_hot(seq):
    f = np.zeros((len(seq), 20), np.float32)
    f[np.arange(len(seq)), seq] = 1.0
    return f


def edge_profile(rng, L):
    return _profile(_dirichlet(rng, L, 0.5), rng.uniform(1.0, 10.0, L), rng.uniform(1.0, 10.0))


def single_sequence(rng, L):
    """The first-iteration query of hhblits: one sequence, one-hot rows, Neff_M = 1."""
    return _profile(_one_hot(rng.integers(0, 20, L)), np.ones(L), 1.0)


def conserved(rng, L):
    """Long identical one-hot windows at high Neff: extreme context scores, almost every exp(ppi[k] - tmp) underflows
    and the posterior is nearly one state."""
    seq = np.empty(L, np.int64)
    pos = 0
    while pos < L:
        n = int(rng.integers(15, 40))
        seq[pos:pos + n] = rng.integers(0, 20) if rng.random() < 0.5 else rng.integers(0, 20, min(n, L - pos))
        pos += n
    return _profile(_one_hot(seq), rng.uniform(12.0, 20.0, L), 18.0)


def diverse(rng, L):
    """Dirichlet rows of small (peaked) and large (flat) concentration, Neff_M across [1, 20]."""
    alpha = np.where(rng.random(L) < 0.5, 0.05, 5.0)
    f = np.stack([rng.dirichlet(np.full(20, a)) for a in alpha]).astype(np.float32)
    return _profile(f, rng.uniform(1.0, 20.0, L), rng.uniform(1.0, 20.0))


def mixed(rng, L):
    """Conserved and diverse runs alternating, with exact zero entries in the diverse rows."""
    f = np.zeros((L, 20), np.float32)
    neff = np.zeros(L)
    pos, cons = 0, bool(rng.integers(0, 2))
    while pos < L:
        n = min(int(rng.integers(5, 30)), L - pos)
        if cons:
            f[pos:pos + n] = _one_hot(np.full(n, rng.integers(0, 20)))
            neff[pos:pos + n] = rng.uniform(1.0, 20.0)
        else:
            d = rng.dirichlet(np.full(20, 0.3), n)
            d[rng.random((n, 20)) < 0.4] = 0.0
            d[np.arange(n), rng.integers(0, 20, n)] += 0.1
            f[pos:pos + n] = (d / d.sum(axis=1, keepdims=True)).astype(np.float32)
            neff[pos:pos + n] = rng.uniform(1.0, 8.0, n)
        pos += n
        cons = not cons
    return _profile(f, neff, rng.uniform(1.0, 12.0))


def long_profile(rng, L):
    """A long query: diverse and conserved stretches (mixed), L up to the query limit."""
    return mixed(rng, L)


def longest_query(L=MAX_QUERY):
    """The seeded query of the query-limit test, made the same way in the test and in the reference's child process."""
    return long_profile(np.random.default_rng([L, 7]), L)


def family(name, seed=0, W=W_DEFAULT):
    """[(tag, (f, neff_m, neff_hmm))] of one count-profile family."""
    rng = np.random.default_rng([seed, sum(map(ord, name)), W])
    if name == "edges":
        return [(f"edges L={L}", edge_profile(rng, L)) for L in edge_lengths(W)]
    if name == "single":
        return [(f"single L={L}", single_sequence(rng, L)) for L in (1, 5, 13, 40, 257)]
    if name == "conserved":
        return [(f"conserved L={L}", conserved(rng, L)) for L in (13, 64, 300)]
    if name == "diverse":
        return [(f"diverse L={L}", diverse(rng, L)) for L in (9, 100, 400)]
    if name == "mixed":
        return [(f"mixed L={L}", mixed(rng, L)) for L in (30, 211, 500)]
    if name == "long":
        return [(f"long L={L}", long_profile(rng, L)) for L in (1500, 4094)]
    raise KeyError(name)


FAMILIES = ("edges", "single", "conserved", "diverse", "mixed", "long")


# --------------------------------------------------------------------------------------------- synthetic context libraries
def crf_text(states, W, names=None):
    """A `.crf` text as cs::Crf::Write + CrfState::Write write it (src/cs/crf-inl.h:79-86, crf_state-inl.h:79-107).
    states: [(bias, w[W][20] of ints or "*", pc[20] ints)]; names[k] or None (no NAME line)."""
    out = ["CRF\n", f"SIZE\t{len(states)}\n", f"LENG\t{W}\n"]
    for k, (bias, w, pc) in enumerate(states):
        out.append("CrfState\n")
        if names is not None and names[k]:
            out.append(f"NAME\t{names[k]}\n")
        out.append("BIAS\t%-10.8g\n" % bias)
        out.append(f"LENG\t{len(w)}\nALPH\t20\n")
        out.append("WEIGHTS" + "".join("\t" + a for a in AA) + "\n")
        for i, row in enumerate(w):
            out.append(str(i + 1) + "".join("\t" + str(v) for v in row) + "\n")
        out.append("PC" + "".join("\t" + str(v) for v in pc) + "\n//\n")
    return "".join(out).encode()


def random_states(rng, K, W, stars=False):
    """K states of window W: biases of both signs, context weights mostly within +-3000 (thousandths) with a few across
    the whole int range, and '*' (the reader's INT_MAX / 1000) when stars is set."""
    states = []
    for _ in range(K):
        w = rng.integers(-3000, 3001, (W, 20)).astype(object)
        wide = rng.random((W, 20)) < 0.01
        w[wide] = rng.integers(-2**31 + 1, 2**31, int(wide.sum()))
        if stars:
            w[rng.random((W, 20)) < 0.005] = "*"
        pc = rng.integers(-4000, 4001, 20)
        states.append((float(rng.normal(-2.0, 3.0)), w.tolist(), pc.tolist()))
    return states


# (K, W, NAME lines, '*' weights): K around k_crf_scores' block of 256 threads, W up to the 63 columns it holds
LIBRARIES = [(1, 1, False, False), (2, 3, True, False), (255, 13, False, True), (256, 15, True, False),
             (257, 63, True, True), (1000, 13, False, False), (1, 63, False, True), (256, 1, True, False)]


def library(K, W, names=False, stars=False, seed=0):
    rng = np.random.default_rng([seed, K, W, int(names), int(stars)])
    nm = [f"state{k}" if rng.random() < 0.7 else "" for k in range(K)] if names else None
    return crf_text(random_states(rng, K, W, stars), W, nm)


def libraries():
    """[(tag, text)] of every synthetic library."""
    return [(f"K={K} W={W}{' names' if n else ''}{' stars' if s else ''}", library(K, W, n, s)) for K, W, n, s in LIBRARIES]


def _edit(text, old, new, count=1):
    assert old in text
    return text.replace(old, new, count)


def refused_by_both():
    """[(tag, text)]: texts the reference's reader and the library's parser both refuse."""
    base = library(3, 5, names=True, seed=7)
    rows = base.split(b"\n")
    return [
        # the trailing line keeps the reader off end-of-file, where it would test a buffer fgets did not fill
        ("SIZE larger than the states given", _edit(base, b"SIZE\t3", b"SIZE\t4") + b"END\n"),
        ("a state with fewer weight rows than LENG", b"\n".join(r for r in rows if not r.startswith(b"5\t"))),
        ("not a CRF", b"CRX\n" + base[4:]),
        ("a state without BIAS", _edit(base, b"BIAS", b"BIOS")),
        ("alphabet size 21", _edit(base, b"ALPH\t20", b"ALPH\t21")),
        ("no states", base[:base.index(b"CrfState")] + b"\nEND\n"),
    ]


def refused_by_library():
    """[(tag, text, reason)]: texts only the library refuses, each a deliberate limit or a text the reference reads
    into undefined state.  Even windows are not given to the reference at all: its reader asserts on them."""
    base = library(3, 5, seed=8)
    no_pc = b"\n".join(r for r in base.split(b"\n") if not r.startswith(b"PC"))
    second = base.index(b"CrfState", base.index(b"CrfState") + 1)
    other_len = base[:second] + crf_text(random_states(np.random.default_rng(9), 1, 7), 7)[len(b"CRF\nSIZE\t1\nLENG\t7\n"):]
    other_len += base[base.index(b"CrfState", second + 1):]
    return [
        ("window 65", library(2, 65, seed=1), "window longer than 63"),
        ("a state without a PC row", no_pc, "the reference keeps uninitialised PC weights"),
        ("a state LENG differing from the CRF's", other_len, "every state's window must be the library's window"),
    ]


def even_window():
    return library(2, 4, seed=2)


# --------------------------------------------------------------------------------------------------------------- goldens
# The comparisons that need a custom library or an admixture other than the two defaults read tests/golden/crf_v1.npz:
# what the reference's hhref_context_pc_crf / hhref_crf_text_state computed on these inputs (tests/golden/
# make_crf_golden.py).  They do not need a compiled reference of this revision, so an oracle/_ref built from an earlier
# revision of oracle/ref_shim.cpp still runs them; the two default engines are compared with the live reference.  Each
# case keeps a digest of its inputs (library text, count profile, admixture), so a generator that drifted fails loudly,
# and one digest per profile row of the reference's p, so a difference names its column.
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "crf_v1.npz")
SYNTH_TAIL = (255, 13, False, True)             # the synthetic library of the CPU tail test
SYNTH_REUSE = (257, 63, True, True)             # the synthetic library of the context-reuse test
REUSE_LENGTHS = (400, 4094, 1, 13, 2000)


def golden():
    return np.load(GOLDEN)


def row_digests(p):
    """One 64-bit digest of the float32 bits of each row of p."""
    p = np.ascontiguousarray(p, np.float32)
    return np.array([int.from_bytes(hashlib.blake2b(r.tobytes(), digest_size=8).digest(), "little") for r in p], np.uint64)


def input_digest(text, f, neff_m, neff_hmm, adm):
    h = hashlib.sha256(hashlib.sha256(text).digest())
    for a in (f, neff_m, np.float32(neff_hmm)):
        h.update(np.ascontiguousarray(a, np.float32).tobytes())
    h.update(repr(tuple(float(x) for x in adm)).encode())
    return np.frombuffer(h.digest(), np.uint8)


def text_digest(text):
    return np.frombuffer(hashlib.sha256(text).digest(), np.uint8)


def state_digest(pc, bias, w):
    """Digest of one parsed state: its pseudocounts, bias and context weights as float64 bits."""
    b = np.ascontiguousarray(pc, np.float64).tobytes() + np.float64(bias).tobytes() + np.ascontiguousarray(w, np.float64).tobytes()
    return int.from_bytes(hashlib.blake2b(b, digest_size=8).digest(), "little")


def tail_profiles():
    return (family("edges")[:4] + family("edges")[-2:] + family("single")[:3] + family("diverse")[:1] +
            family("conserved")[:1])


def golden_cases(embedded):
    """{group: [(key, text, adm, (f, neff_m, neff_hmm))]} of every pseudocount case the goldens hold; embedded is the
    text of the reference's context_data.crf (RefShim.crf_text())."""
    out = dict(tail=[], admix=[], lib=[], reuse=[])
    synth = library(*SYNTH_TAIL)
    for ai, adm in enumerate(ADMIXTURES):
        for lt, text, profiles in (("embedded", embedded, tail_profiles()), ("K=255 W=13 stars", synth, family("diverse")[:2])):
            out["tail"] += [(f"tail/{ai}/{lt}/{tag}", text, adm, prof) for tag, prof in profiles]
        for fam in ("edges", "single", "diverse"):
            out["admix"] += [(f"admix/{ai}/{tag}", embedded, adm, prof) for tag, prof in family(fam, seed=1)]
    for lt, text in libraries():
        W = int(text.split(b"\n")[2].split(b"\t")[1])
        rng = np.random.default_rng(400)
        cases = family("edges", W=W) + [("diverse L=400", diverse(rng, 400))]
        out["lib"] += [(f"lib/{lt}/{tag}", text, (ADMIX_HHM, ADMIX_PREFILTER)[k % 2], prof)
                       for k, (tag, prof) in enumerate(cases)]
    profiles = reuse_profiles()
    out["reuse"] = [(f"reuse/L={L}", library(*SYNTH_REUSE), ADMIX_PREFILTER, profiles[L]) for L in REUSE_LENGTHS]
    return out


def reuse_profiles():
    """The count profiles of the context-reuse test, by length."""
    rng = np.random.default_rng(4094)
    return {L: mixed(rng, L) for L in REUSE_LENGTHS}


def expected(G, key, text, adm, prof):
    """(row digests, pav) the reference computed for this case, after checking the golden holds these very inputs."""
    f, neff_m, neff_hmm = prof
    assert f"h/{key}" in G.files, f"no golden for {key}"
    assert np.array_equal(G[f"h/{key}"], input_digest(text, f, neff_m, neff_hmm, adm)), \
        f"the inputs of {key} are not those tests/golden/crf_v1.npz was made from"
    return G[f"d/{key}"], G[f"pav/{key}"]


def compare(got_p, got_pav, want, tag, rows=None):
    """got (p, pav) against expected(): the first differing column is named; rows limits the comparison (the host
    tail fills rows 1..L only), got_pav None skips pav."""
    digests, pav = want
    d = row_digests(got_p)
    sel = slice(None) if rows is None else rows
    bad = np.flatnonzero(d[sel] != digests[sel])
    assert len(bad) == 0, (tag, f"{len(bad)} columns differ from the reference, the first is column "
                           f"{int(bad[0]) + (0 if rows is None else rows.start)}")
    assert got_pav is None or np.array_equal(np.asarray(got_pav, np.float32).view(np.uint32), pav.view(np.uint32)), (tag, "pav")
