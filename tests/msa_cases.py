"""Synthetic A3M alignments shared by the alignment -> HMM tests (CPU scanner test and GPU parity tests), and the seeded
random generators of the randomised tests and tools/msa_fuzz.py."""
import os

import numpy as np

CASES = [  # (match columns, sequences after the master, seed, generator options)
    (50, 20, 1, {}),
    (8, 5, 2, {}),                                    # fewer than NCOLMIN columns: global weights everywhere
    (120, 300, 3, dict(with_ss=True)),
    (200, 60, 4, dict(with_comment=True)),
    (80, 40, 5, dict(consensus_first=True)),          # compressed databases: consensus row outside the profile
    (30, 0, 6, {}),                                   # single sequence
    (300, 150, 7, dict(ident=0.9, dup_frac=0.6)),     # most rows removed by the 90 % identity filter
    (15, 3, 8, dict(with_ss=True, with_comment=True)),
    (60, 1, 9, {}),
    (431, 58, 10, dict(ident=0.3)),
    (700, 90, 11, dict(ident=0.6, with_ss=True)),
    (90, 25, 12, dict(with_ss=True, ss_conf=False)),  # ss_pred without ss_conf: confidence 5 everywhere
]


# hand-written corner cases (CPU tests): a single sequence with fewer than six match states falls back to "-M first"
# (src/hhalignment.cpp:861-880): lower-case letters become match states, '-' columns do not
TINY = [b">master\nZ-iwHkv\n", b"#NAME some description\n>master\nlKV\n", b">ss_pred\nHHEC-\n>ss_conf\n12345\n>m\nAc-dE\n",
        b">m\r\nACDEFGHIKL\r\n>s1 x\r\nAC-EFGHIKL\r\n>s2\r\n.ACDEFGaaHIKL\r\n"]


# (text, M, Mgaps, filter (max_seqid, coverage, qid, qsc, Ndiff)) under the -M <percent> / -M first rules.  The first:
# Compress moves the match columns to the front of each row in place, and Filter2's 32-byte windows count the input
# columns it left past column L; with them the reference rejects s3, without them s3 passes the filter.
MRULE_CASES = [
    (b">master\nGHSMRXQDXVMNSHMVFQNFCQX-RaQKLVYME\n>s0\n-NTKXK-iHMDFMCXN-SX-IfGPDSMFEFNCM\n"
     b">s1\n--INPQ-RAICSMT--XFPRAKHPDDHTKDPFS\n>s2\n-CPYDVLLI-FKE-HYKLP-VSDg-YELSGF-S\n"
     b">s3\nXIT--Q-HGXFDSLQYKLTQSPCQLHVNTFCF-\n>s4\n-MXEVCYLR-WR-ET-GLK-APAQLWVDSDMKQ\n"
     b">s5\n-PWHLT-E-PE-NLSXAV--F-dAIQ-PNAPYK\n>s6\n-FGG-H-Q-CSWDHaRFLP-IXMAIE-ITKRNG\n"
     b">s9\n--HGNCWA--QXSANDGLSWgXPEQNMRGXThF\n>s19\n-RCGNFDA-CYILIQ-ICS-RITH-AMKDRYYV\n"
     b">s34\n-YPDEGYV-QFSXHIKLFL-NYE-FWKKVNMYL\n", 2, 50, (90, 0, 0, -20.0, 10)),
]


def texts():
    from hhsuite_b200 import synth
    out = [synth.a3m_text(L, n, seed, **kw).encode() for (L, n, seed, kw) in CASES]
    q = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "oracle", "_ref", "data", "query.a3m")
    if os.path.exists(q):
        out.append(open(q, "rb").read())
    return out


CA3M_CASES = [(50, 20, 21, {}), (120, 200, 22, dict(ident=0.8, dup_frac=0.5)), (300, 40, 23, {}),
              (260, 30, 25, dict(ident=0.4)), (9, 6, 26, {})]


def ca3m_database(directory, alignments=None):
    """A compressed alignment database (<dir>/db_ca3m|_sequence|_header .ffdata/.ffindex) made from synthetic
    alignments: the CA3M_CASES, or the given (name, A3M text) pairs (see ca3m_source).  Returns the prefix."""
    from hhsuite_b200 import ffindex, synth
    prefix = os.path.join(str(directory), "db")
    if alignments is None:
        alignments = [(f"al{seed}", synth.a3m_text(L, n, seed, name=f"al{seed}", **kw)) for (L, n, seed, kw) in CA3M_CASES]
    recs, seqs, heads = [], [], []
    for name, a in alignments:
        ca, sq, hd = synth.a3m_to_ca3m(a, seq_index_base=len(seqs))
        recs.append((name, ca)); seqs += sq; heads += hd
    names = [f"s{i:06d}" for i in range(len(seqs))]
    ffindex.write_ffindex(prefix + "_ca3m.ffdata", recs)
    ffindex.write_ffindex(prefix + "_sequence.ffdata", list(zip(names, seqs)))
    ffindex.write_ffindex(prefix + "_header.ffdata", list(zip(names, heads)))
    return prefix


# ---------------------------------------------------------------------------------------------- seeded random alignments
AA = "ARNDCQEGHILKMFPSTWYV"
MAXROW = 4000        # characters per row, inserts included: the reference is run with maxres = 4096


def rand_a3m(rng, L=None, n=None):
    """A small free-form A3M record: the extended alphabet (X B Z U J O), '-' and '.', insert runs before, inside and
    after the match columns, '#' and ss rows, a '_consensus' master, rows split over two lines and CRLF line ends."""
    L = int(rng.integers(1, 40)) if L is None else L
    n = int(rng.integers(0, 12)) if n is None else n
    alpha = AA + "XBZUJO"
    lines = []
    if rng.random() < 0.3:
        lines.append("#NAME some description")
    if rng.random() < 0.3:
        lines += [">ss_pred", "".join(rng.choice(list("HEC-"), L))]
        if rng.random() < 0.6:
            lines += [">ss_conf", "".join(rng.choice(list("0123456789"), L))]

    def row(first=False):
        out = []
        if rng.random() < 0.2:
            out.append("".join(rng.choice(list(AA.lower()), int(rng.integers(1, 4)))))
        for _ in range(L):
            out.append(rng.choice(list(alpha)) if rng.random() < 0.85 or first else "-")
            if rng.random() < 0.1:
                out.append("".join(rng.choice(list(AA.lower()), int(rng.integers(1, 4)))))
            if rng.random() < 0.03:
                out.append(".")
        s = "".join(out)
        return s if any(ch.isalpha() for ch in s) else "A" + s[1:]
    lines += [">master" if rng.random() < 0.9 else ">cons_consensus", row(True)]
    for k in range(n):
        lines.append(f">s{k}")
        s = row()
        if rng.random() < 0.3 and len(s) > 4:
            c = int(rng.integers(1, len(s) - 1)); lines += [s[:c], s[c:]]
        else:
            lines.append(s)
    eol = "\r\n" if rng.random() < 0.2 else "\n"
    return (eol.join(lines) + eol).encode()


def rand_fasta(rng, L=None, n=None):
    """An aligned-FASTA record (every row has all columns; '-' gaps, gap-rich columns, a few lower-case residues) for
    the -M <percent> and -M first rules."""
    L = int(rng.integers(3, 60)) if L is None else L
    n = int(rng.integers(1, 15)) if n is None else n
    pg = np.where(rng.random(L) < 0.25, 0.7, 0.08)
    alpha = np.array(list(AA + "X"))
    lines = []
    for k in range(n + 1):
        gap = rng.random(L) < pg
        if k == 0:
            gap &= rng.random(L) >= 0.5
        res = alpha[rng.integers(0, len(alpha), L)]
        res = np.where(rng.random(L) < 0.05, np.char.lower(res), res)
        s = "".join(np.where(gap, "-", res))
        lines += [">master" if k == 0 else f">s{k - 1}", s if any(ch.isalpha() for ch in s) else "A" + s[1:]]
    return ("\n".join(lines) + "\n").encode()


def _entries(text):
    """[header, sequence] of an A3M text (rows joined); '#' lines are entries without a sequence."""
    out = []
    for ln in text.splitlines():
        if ln.startswith("#") or ln.startswith(">"):
            out.append([ln, None if ln.startswith("#") else ""])
        else:
            out[-1][1] += ln
    return out


def _text(entries, rng, crlf=0.0, wrap=0.0):
    lines = []
    for h, s in entries:
        lines.append(h)
        if s is None:
            continue
        if rng.random() < wrap and len(s) > 1:
            w = int(rng.integers(1, 120))
            lines += [s[i:i + w] for i in range(0, len(s), w)]
        else:
            lines.append(s)
    eol = "\r\n" if rng.random() < crlf else "\n"
    return eol.join(lines) + eol


def _edit_rows(entries, fn):
    """fn(k, [(match char, insert run after it)], lead insert) -> (match chars, inserts, lead) for every sequence after
    the master (entries k >= 1 of the profile rows)."""
    rows = [e for e in entries if e[1] is not None and not e[0].startswith((">ss_", ">sa_"))]
    for k, e in enumerate(rows[1:]):
        s = e[1]
        lead = ""
        cols = []
        for c in s:
            if c.isupper() or c == "-":
                cols.append([c, ""])
            elif cols:
                cols[-1][1] += c
            else:
                lead += c
        cols, lead = fn(k, cols, lead)
        s = lead + "".join(c + i for c, i in cols)
        if not any(ch.isalpha() for ch in s):
            s = "A" + s[1:]
        e[1] = s


def _master_only(rng, L):
    """Columns at which only the master has a residue (runs of them)."""
    J = np.zeros(L, bool)
    for _ in range(int(rng.integers(1, 6))):
        a = int(rng.integers(0, L)); J[a:a + int(rng.integers(1, max(2, L // 6)))] = True
    return lambda k, cols, lead: ([["-" if J[j] else c, "" if J[j] else i] for j, (c, i) in enumerate(cols)], lead)


def _short_window(rng, L):
    """Every row cut down to a short window of columns: the set of rows with a residue changes at many columns."""
    def fn(k, cols, lead):
        a = int(rng.integers(0, L)); b = min(L, a + int(rng.integers(1, max(2, L // 5))))
        out = [[c, i] if a <= j < b else ["-", ""] for j, (c, i) in enumerate(cols)]
        if all(c == "-" for c, _ in out[a:b]):
            out[a][0] = "A"
        return out, ""
    return fn


def _long_inserts(rng, L):
    def fn(k, cols, lead):
        if rng.random() < 0.6:
            for _ in range(int(rng.integers(1, 4))):
                j = int(rng.integers(0, L))
                cols[j][1] += "".join(rng.choice(list(AA.lower()), int(rng.integers(20, 150))))
        return cols, lead
    return fn


FAMILIES = ("tiny", "typical", "long", "deep", "master_only", "short_window", "identical", "long_inserts")


def _draw(rng, family):
    from hhsuite_b200 import synth
    seed = int(rng.integers(1, 2 ** 31))
    ss = rng.random() < 0.3
    kw = dict(with_ss=ss, ss_conf=bool(rng.random() < 0.6), with_comment=bool(rng.random() < 0.3),
              ident=float(rng.uniform(0.3, 0.97)), dup_frac=float(rng.uniform(0, 0.7)))
    logu = lambda lo, hi: int(round(np.exp(rng.uniform(np.log(lo), np.log(hi)))))  # noqa: E731
    if family == "tiny":
        L, n = int(rng.integers(1, 13)), int(rng.integers(0, 6))
        u = rng.random()
        if u < 0.2:        # one sequence of fewer than six match states: read with -M first semantics
            return rand_a3m(rng, int(rng.integers(1, 6)), 0).decode()
        if u < 0.5:
            return rand_a3m(rng, L, n).decode()
        return _text(_entries(synth.a3m_text(L, n, seed, **kw)), rng, crlf=0.2, wrap=0.2)
    if family == "typical":
        kw["consensus_first"] = bool(rng.random() < 0.1)
        return _text(_entries(synth.a3m_text(logu(30, 400), logu(5, 300), seed, **kw)), rng, crlf=0.2, wrap=0.3)
    if family == "long":
        return synth.a3m_text(int(rng.integers(1500, 3001)), int(rng.integers(20, 81)), seed,
                              with_ss=ss, ident=float(rng.uniform(0.3, 0.9)))
    if family == "deep":
        return synth.a3m_text(int(rng.integers(60, 151)), int(rng.integers(1500, 3001)), seed,
                              ident=float(rng.uniform(0.3, 0.9)), dup_frac=float(rng.uniform(0, 0.5)))
    L, n = logu(20, 300), logu(2, 120)
    e = _entries(synth.a3m_text(L, n, seed, **kw))
    if family == "identical":             # every row is the master: the filter keeps one row
        m = next(s for h, s in e if s is not None and not h.startswith(">ss_"))
        for x in e[1:]:
            if x[1] is not None and not x[0].startswith(">ss_"):
                x[1] = m
    else:
        _edit_rows(e, dict(master_only=_master_only, short_window=_short_window, long_inserts=_long_inserts)[family](rng, L))
    return _text(e, rng, crlf=0.1, wrap=0.2)


def accepted(text, M=1, Mgaps=50):
    """True if the library's host scanner takes the record (it refuses exactly what makes the reference exit)."""
    from hhsuite_b200 import capi
    try:
        capi.a3m_parse(text, capi.MsaParams.defaults(M=M, Mgaps=Mgaps))
    except capi.HhgError:
        return False
    return max(len(s) for h, s in _entries(text.decode()) if s is not None) < MAXROW


def random_alignment(rng, family):
    """One seeded A3M record (bytes) of a shape family (FAMILIES) that the reference accepts."""
    for _ in range(20):
        t = _draw(rng, family).encode()
        if accepted(t):
            return t
    raise RuntimeError(f"no acceptable {family} alignment in 20 draws")


def ca3m_source(rng, family):
    """A random_alignment of the family in the form synth.a3m_to_ca3m compresses (no ss rows, no '.', a master and at
    least one more sequence); the master becomes the record's consensus row."""
    for _ in range(20):
        e = [x for x in _entries(random_alignment(rng, family).decode()) if not x[0].startswith((">ss_", ">sa_"))]
        rows = [s for h, s in e if s is not None]
        if len(rows) >= 2 and not any("." in s for s in rows):
            return _text(e, rng, wrap=0.2)
    raise RuntimeError(f"no {family} alignment for a compressed record in 20 draws")


def random_fasta(rng, M, Mgaps=50):
    """An aligned-FASTA record of typical size (30..400 columns, 5..300 sequences) for -M <percent> / -M first."""
    for _ in range(20):
        L = int(round(np.exp(rng.uniform(np.log(30), np.log(400)))))
        t = rand_fasta(rng, L, int(round(np.exp(rng.uniform(np.log(5), np.log(300))))))
        if accepted(t, M, Mgaps):
            return t
    raise RuntimeError("no acceptable aligned-FASTA record in 20 draws")


def random_filter(rng):
    """(max_seqid, coverage, qid, qsc, Ndiff) and wg drawn like tools/msa_fuzz.py."""
    filt = (int(rng.choice([15, 40, 60, 75, 90, 95, 100])), int(rng.choice([0, 0, 20, 50, 80])),
            int(rng.choice([0, 0, 15, 30, 50])), float(rng.choice([-20.0, -20.0, 0.0, 0.3])), int(rng.choice([0, 3, 5, 10, 100])))
    return filt, int(rng.random() < 0.3)
