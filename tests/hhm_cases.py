"""Seeded HHM record families shared by the HHM loader tests (CPU: oracle and tokeniser against the compiled reference;
GPU: the resident, staged and query loaders).  Each generator takes (seed, L) and returns the bytes of one record.

  hhmake    the layout HMM::WriteToFile produces (src/hhhmm.cpp:2173-2299): '*' emissions from small counts, one-hot and
            all-'*' columns, Neff_I / Neff_D of 0 with '*' transitions, MSA column indices that are not i, a SEQ block
            with ss_dssp / sa_dssp / ss_pred / ss_conf / Consensus and up to 10 sequences wrapped at 100 characters
  variants  header and syntax forms HMM::Read accepts: NAA, 'NEFF x' with one space, EVD / DESC, CRLF, trailing blanks,
            blank lines or none between columns, skipped column numbers, consensus '-' / 'X', negative integers, odd
            ss_pred letters, ss_conf before ss_pred, a second ss_pred, ss_pred or ss_conf alone, an empty SEQ block, no
            newline after '//', an ffindex NUL and garbage after the record
  values    numeric edges: Neff_M 0 and '*', Neff_I / Neff_D 0 and 99999, transitions 0 and '*', PCT, NULL lines with 0
            and '*', L = 1, 2, 3 and 4k + r for every r
  sweep     sweep_records(): emission, transition and Neff integers that together take every value 0..99999 and '*'
  written   written(): records the reference's own writer produced from seeded alignments (needs the compiled reference)

Every family keeps the standard NULL line (synth._NULL_MILLIBITS) unless stated: values() writes other NULL lines when
null=True, and a test that reads such a record with the compiled reference must put the reference's pb back.

NAMED_CASES are the divergences these families found, one record each (see the tests that use them)."""
import numpy as np

AA_SORTED = "ACDEFGHIKLMNPQRSTVWY"
STAR = 1_000_000             # written as '*', which strinta reads as 99999 (src/util.cpp:175)
MAXREF = 4094                # longest record the compiled reference reads with maxres = 4096


def _null_std():
    from hhsuite_b200 import synth
    return [int(v) for v in synth._NULL_MILLIBITS]


def _num(v):
    return "*" if v == STAR else str(int(v))


def _wrap(s, w=100):
    return [s[k:k + w] for k in range(0, len(s), w)] or [""]


def _counts_columns(rng, L):
    """Emission integers from small integer counts (what hhmake writes for shallow alignments): many '*', one-hot
    columns (one 0, 19 '*') and all-'*' columns."""
    f = np.full((L, 20), STAR, np.int64)
    for i in range(L):
        kind = rng.random()
        if kind < 0.12:
            f[i, int(rng.integers(0, 20))] = 0
        elif kind < 0.18:
            pass                                                    # all '*'
        else:
            n = int(rng.integers(1, 12))
            c = rng.multinomial(n, rng.dirichlet(np.full(20, 0.3)))
            with np.errstate(divide="ignore"):
                x = np.round(-1000.0 * np.log2(c / n))
            f[i] = np.where(c > 0, x, STAR).astype(np.int64)
    return f


def _transitions(rng, L, zero_frac=0.4):
    """Transition integers (M->M, M->I, M->D, I->M, I->I, D->M, D->D) and Neff_M, Neff_I, Neff_D * 1000 for rows 0..L:
    Neff_I / Neff_D often 0 with '*' on the transitions they govern."""
    tr = rng.integers(0, 6000, (L + 1, 7)).astype(np.int64)
    ne = np.stack([rng.integers(1000, 12000, L + 1), rng.integers(0, 5000, L + 1), rng.integers(0, 5000, L + 1)], 1)
    for i in range(L + 1):
        if rng.random() < zero_frac:
            ne[i, 1] = 0; tr[i, 3] = 0; tr[i, 4] = STAR
        if rng.random() < zero_frac:
            ne[i, 2] = 0; tr[i, 5] = 0; tr[i, 6] = STAR
        if rng.random() < 0.3:
            tr[i, 0] = 0; tr[i, 1] = STAR; tr[i, 2] = STAR
    tr[0] = [0, STAR, STAR, 0, STAR, 0, STAR]                      # hhmake's start row
    return tr, ne.astype(np.int64)


def _ss_rows(rng, L):
    pred = "".join(rng.choice(list("HEC"), L))
    conf = "".join(str(d) for d in rng.integers(0, 10, L))
    dssp = "".join(rng.choice(list("HEC-STGB"), L))
    sa = "".join(rng.choice(list("ABCDE-"), L))
    return pred, conf, dssp, sa


def compose(L, f, tr, ne, *, null=None, head=None, seq=None, cons=None, colnum=None, lidx=None, eol="\n",
            gap_lines=True, trail="\t", pct=False, neff_line=None, end="//\n", start_row_neff=None):
    """Write one HHM record from its integers; every keyword changes one feature of the layout."""
    null = _null_std() if null is None else null
    cons = cons if cons is not None else "".join(AA_SORTED[int(np.argmin(r))] for r in f)
    colnum = colnum if colnum is not None else list(range(1, L + 1))
    lidx = lidx if lidx is not None else list(range(1, L + 1))
    out = ["HHsearch 1.5"]
    out += head if head is not None else ["NAME  case", "FAM   ", f"LENG  {L} match states, {L} columns in multiple alignment",
                                          "FILT  1 out of 1 sequences passed filter"]
    out.append(neff_line if neff_line is not None else "NEFF  3.0 ")
    if pct:
        out.append("PCT   true")
    out.append("SEQ")
    out += seq if seq is not None else [">Consensus", cons.lower(), ">case", cons]
    out.append("#")
    out.append("NULL   " + "\t".join(_num(v) for v in null) + trail)
    out.append("HMM    " + "\t".join(AA_SORTED) + "\t")
    out.append("       M->M\tM->I\tM->D\tI->M\tI->I\tD->M\tD->D\tNeff\tNeff_I\tNeff_D")
    r0 = start_row_neff if start_row_neff is not None else ne[0]
    out.append("       " + "\t".join(_num(v) for v in tr[0]) + "\t" + "\t".join(_num(v) for v in r0) + trail)
    for i in range(1, L + 1):
        out.append(f"{cons[i - 1]} {colnum[i - 1]:<4d} " + "\t".join(_num(v) for v in f[i - 1]) + f"\t{lidx[i - 1]}" + trail)
        out.append("       " + "\t".join(_num(v) for v in tr[i]) + "\t" + "\t".join(_num(v) for v in ne[i]) + trail)
        if gap_lines:
            out.append("")
    return (eol.join(out) + eol + end.replace("\n", eol)).encode()


# ------------------------------------------------------------------------------------------------------------- hhmake
def hhmake(seed, L):
    rng = np.random.default_rng(seed)
    f = _counts_columns(rng, L)
    tr, ne = _transitions(rng, L)
    lidx = list(np.cumsum(rng.integers(1, 4, L)))                  # MSA column indices l[i]: inserts skipped
    pred, conf, dssp, sa = _ss_rows(rng, L)
    cons = "".join(AA_SORTED[int(rng.integers(0, 20))] for _ in range(L))
    rows = [(">ss_dssp", dssp), (">sa_dssp", sa), (">ss_pred PSIPRED predicted secondary structure", pred),
            (">ss_conf PSIPRED confidence values", conf), (">Consensus", cons.lower())]
    keep = [r for r in rows if rng.random() < 0.6]
    if rng.random() < 0.5:
        rng.shuffle(keep)
    for k in range(int(rng.integers(1, 11))):
        s = "".join(rng.choice(list(AA_SORTED + "-"), L))
        keep.append((f">seq{k} sequence {k} of an alignment", s))
    seq = []
    for h, s in keep:
        seq += [h] + _wrap(s)
    neff = float(rng.uniform(1.0, 14.0))
    head = [f"NAME  fam{seed} a protein family description", "FAM   a.1.1.1",
            "COM   hhmake -i " + "/data/alignments/" * 8 + f"fam{seed}.a3m -o fam{seed}.hhm -M first",
            "DATE  Fri Oct 16 00:00:00 2026", f"LENG  {L} match states, {int(lidx[-1])} columns in multiple alignment", "",
            f"FILT  {int(rng.integers(1, 99))} out of 100 sequences passed filter (-id 90 -cov 0 -qid 0 -qsc -20 -diff 100)"]
    return compose(L, f, tr, ne, head=head, seq=seq, cons=cons, lidx=lidx, neff_line=f"NEFF  {neff:<4.1f}")


# ----------------------------------------------------------------------------------------------------------- variants
VARIANTS = ("naa", "neff_one_space", "evd_desc", "crlf", "trailing_blanks", "no_gap_lines", "skipped_colnums",
            "consensus_dash_x", "negative_ints", "ss_odd_letters", "conf_before_pred", "second_pred", "pred_only",
            "conf_only", "empty_seq", "no_final_newline", "nul_garbage")


def variants(seed, L):
    """A record with two or three of the VARIANTS features (chosen by the seed; VARIANTS[seed % n] always)."""
    rng = np.random.default_rng(seed)
    feats = {VARIANTS[seed % len(VARIANTS)]} | {str(x) for x in rng.choice(VARIANTS, 2, replace=False)}
    return variant(seed, L, feats)


def variant(seed, L, feats):
    rng = np.random.default_rng(10_000 + seed)
    f = _counts_columns(rng, L)
    tr, ne = _transitions(rng, L)
    pred, conf, _, _ = _ss_rows(rng, L)
    kw = {}
    neff = f"{rng.uniform(1.0, 14.0):.1f}"
    kw["neff_line"] = f"NEFF  {neff}"
    if "naa" in feats:
        kw["neff_line"] = f"NAA   {neff}"
    if "neff_one_space" in feats:
        kw["neff_line"] = f"NEFF 1{neff}"                         # read from offset 6: the value without its first digit
    head = ["NAME  var", "FAM   ", f"LENG  {L} match states, {L} columns in multiple alignment"]
    if "evd_desc" in feats:
        head += ["EVD   0.2561 -12.3041", "DESC  a description line"]
    kw["head"] = head
    if "crlf" in feats:
        kw["eol"] = "\r\n"
    kw["trail"] = " \t " if "trailing_blanks" in feats else "\t"
    if "no_gap_lines" in feats:
        kw["gap_lines"] = False
    if "skipped_colnums" in feats:
        kw["colnum"] = list(np.cumsum(rng.integers(1, 3, L)))      # HMM::Read only warns
    cons = "".join(AA_SORTED[int(rng.integers(0, 20))] for _ in range(L))
    if "consensus_dash_x" in feats:
        cons = "".join(rng.choice(list("-X" + AA_SORTED[:3]), L))
    kw["cons"] = cons
    if "negative_ints" in feats:
        for _ in range(max(1, L // 3)):
            f[int(rng.integers(0, L)), int(rng.integers(0, 20))] = -int(rng.integers(1, 900))
            tr[int(rng.integers(1, L + 1)), int(rng.integers(0, 7))] = -int(rng.integers(1, 900))
    seq = [">Consensus", cons.lower()]
    pred_lines = [">ss_pred"] + _wrap(pred, 37)
    conf_lines = [">ss_conf"] + _wrap(conf, 37)
    if "ss_odd_letters" in feats:
        odd = "h~ISTGB.Qc-xei" + "".join(rng.choice(list("HECheclowercase~ISTGB.-xQ"), L + L // 4))
        pred_lines = [">ss_pred"] + _wrap(odd, 50)
        conf_lines = [">ss_conf"] + _wrap("".join(rng.choice(list("0123456789-.,"), L + 5)), 50)
    if "conf_only" in feats:
        seq += conf_lines
    elif "pred_only" in feats:
        seq += pred_lines
    elif "conf_before_pred" in feats:
        seq += conf_lines + pred_lines
    elif "second_pred" in feats:
        second = "".join(rng.choice(list("HEC"), max(1, L // 2)))
        seq += pred_lines + conf_lines + [">ss_pred second"] + _wrap(second)
    elif "ss_odd_letters" in feats or rng.random() < 0.5:
        seq += pred_lines + conf_lines
    seq += [">var", cons]
    if "empty_seq" in feats:
        seq = []
    kw["seq"] = seq
    text = compose(L, f, tr, ne, **kw)
    if "no_final_newline" in feats:
        text = text.rstrip(b"\r\n")
    if "nul_garbage" in feats:
        text += b"\0NAME  garbage\nLENG 7\nHMM junk\n"
    return text


# ------------------------------------------------------------------------------------------------------------- values
def values(seed, L, null=False):
    """Numeric edges; null=True also writes a NULL line with 0 and '*' (a non-standard background)."""
    rng = np.random.default_rng(20_000 + seed)
    f = _counts_columns(rng, L)
    tr, ne = _transitions(rng, L, zero_frac=0.3)
    for i in range(L + 1):
        r = rng.random()
        if r < 0.15:
            ne[i, 0] = 0                                            # Neff_M 0 -> 1 (src/hhhmm.cpp:631-633)
        elif r < 0.25:
            ne[i, 0] = STAR                                         # 99.999
        if rng.random() < 0.2:
            ne[i, 1:] = rng.choice([0, STAR, 99999], 2)
        if rng.random() < 0.2:
            tr[i, int(rng.integers(0, 7))] = rng.choice([0, STAR])
    nl = _null_std()
    if null:
        nl[int(rng.integers(0, 20))] = 0
        nl[int(rng.integers(0, 20))] = STAR
    return compose(L, f, tr, ne, null=nl, pct=bool(seed % 2), neff_line=f"NEFF  {rng.uniform(0.1, 20):.1f}")


VALUE_LENGTHS = [1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11, 12, 13, 17, 30, 63]


# -------------------------------------------------------------------------------------------------------------- sweep
def sweep_records(seed=0, max_cols=MAXREF):
    """Records whose emission integers take every value 0..99999 and '*', and whose transition and Neff integers (ten
    per row) do the same; no record is longer than max_cols.  With pcm 0 (or PCT) p = fpow2(-x/1000), with gapb 0
    tr = -x/1000: the device's integer -> float conversions and fpow2 over their whole input domain."""
    rng = np.random.default_rng(30_000 + seed)
    dom = np.concatenate([np.arange(100000), [STAR]]).astype(np.int64)
    rows_needed = -(-len(dom) // 10)                               # transition rows 0..L of all records
    nrec = -(-rows_needed // max_cols)
    total_cols = rows_needed - nrec + 1
    lens = [total_cols // nrec + (1 if k < total_cols % nrec else 0) for k in range(nrec)]
    em = np.resize(rng.permutation(dom), total_cols * 20).reshape(total_cols, 20)
    trn = np.resize(rng.permutation(dom), (total_cols + nrec) * 10).reshape(total_cols + nrec, 10)
    out, c, r = [], 0, 0
    for L in lens:
        rows = trn[r:r + L + 1]
        out.append(compose(L, em[c:c + L], rows[:, :7], rows[:, 7:], pct=False, neff_line="NEFF  5.5"))
        c += L; r += L + 1
    return out


# ------------------------------------------------------------------------------------------------------------ written
def written(refshim, seed, L, tmp_dir, add_pc=False):
    """hhmake (the reference's HMM::WriteToFile) on a seeded alignment; add_pc: with nocontxt pseudocounts (PCT)."""
    import os
    from hhsuite_b200 import synth
    rng = np.random.default_rng(40_000 + seed)
    a3m = synth.a3m_text(L, int(rng.integers(0, 40)), 40_000 + seed, name=f"w{seed}", with_ss=bool(seed % 2),
                         ss_conf=seed % 4 != 3, ident=float(rng.uniform(0.3, 0.9)))
    path = os.path.join(str(tmp_dir), f"w{seed}.a3m")
    with open(path, "w") as fh:
        fh.write(a3m)
    return refshim.write_hhm(path, add_pc)


# --------------------------------------------------------------------------------------------------- family registry
def family(name, n=6, seed0=0):
    """n records of a generated family (not 'written' or 'sweep'): (seed, L, text) with small L and the family's
    length rules."""
    out = []
    for k in range(n):
        s = seed0 + k
        if name == "hhmake":
            L = int(np.random.default_rng(s).integers(1, 300))
            out.append((s, L, hhmake(s, L)))
        elif name == "variants":
            L = int(np.random.default_rng(s).integers(1, 200))
            out.append((s, L, variants(s, L)))
        elif name == "values":
            L = VALUE_LENGTHS[s % len(VALUE_LENGTHS)]
            out.append((s, L, values(s, L)))
        else:
            raise KeyError(name)
    return out


FAMILIES = ("hhmake", "variants", "values")


# ------------------------------------------------------------------------------------------------------- named cases
def _plain(L=20, seed=7, **kw):
    rng = np.random.default_rng(seed)
    f = _counts_columns(rng, L)
    tr, ne = _transitions(rng, L)
    return compose(L, f, tr, ne, **kw)


NAMED_CASES = {
    # HMM::Read takes Neff_HMM from an NAA line as from a NEFF line (src/hhhmm.cpp:296); the tokeniser and the oracle
    # read only NEFF, which left Neff_HMM = 0 and pav NaN for such records
    "naa_line": _plain(neff_line="NAA   4.7"),
    # no NEFF / NAA line: Neff_HMM = 0, pav = pb*100/0 -> NaN in the reference; the loaders refuse the record
    "no_neff": _plain(neff_line="FILT  1 out of 1 sequences passed filter"),
    "neff_zero": _plain(neff_line="NEFF  0.0"),
    # a NEFF line without a number leaves the earlier value (sscanf fails); the tokeniser used to write 0
    "neff_then_empty_neff": _plain(neff_line="NEFF  6.2\nNEFF  n/a"),
    # ss_conf without ss_pred: no secondary structure (ss 0), as records without ss_pred in the same shard
    "conf_only": _plain(seq=[">ss_conf", "1234567890" * 2, ">c", "A" * 20]),
    # ss_pred without ss_conf: the reference leaves ss_conf unset; the loaders write confidence 0
    "pred_only": _plain(seq=[">ss_pred", "HEC" * 6 + "HE", ">c", "A" * 20]),
}


# ------------------------------------------------------------------------------------------- where the reference's ss is set
def _pred_letter(c):
    """HMM::Read stores an ss_pred letter (src/hhhmm.cpp:392-410): ss2i in 0..3, not '.', and ss2ss upper case."""
    u = c.upper()
    code = 0 if u in ".-X" else 1 if u == "H" else 2 if u == "E" else 3 if u in "C~I" else -1
    if code < 0 or c == ".":
        return False
    s = {"~": "C", "I": "C", "i": "c"}.get(c, c if c in "HECSTGBhecstgb." else "-")
    return s != "." and not s.islower()


def ss_defined(text):
    """(n_pred, n_conf): HMM::Read sets ss_pred[1..n_pred] and ss_conf[1..n_conf] of this record and leaves the rest
    of its arrays as they were (uninitialised in a fresh HMM); the loaders write 0 there."""
    npred = nconf = n = 0
    cur, in_seq = None, False
    for line in text.split(b"\0")[0].replace(b"\r", b"").split(b"\n"):
        if not in_seq:
            in_seq = line.startswith(b"SEQ")
            continue
        if line.startswith(b"#"):
            break
        if line.startswith(b">"):
            cur = "p" if line.startswith(b">ss_pred") else "c" if line.startswith(b">ss_conf") else None
            n = 0
            continue
        for c in line.decode("latin1"):
            if cur == "p" and _pred_letter(c):
                n += 1; npred = max(npred, n)
            elif cur == "c" and (c == "-" or c.isdigit()):
                n += 1; nconf = max(nconf, n)
    return npred, nconf
