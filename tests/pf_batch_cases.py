"""Seeded cases of the query-batch prefilter shared by its CPU-emulation and GPU tests (not product code)."""
import numpy as np


def carry_batch(seed, lens=(1700, 1100, 700, 300, 90)):
    """Profiles whose background lies below the offset (every off-diagonal cell decays to 0) with one planted diagonal
    per tile boundary of the query (positions 512, 1024, 1536 where they exist) that gains exactly 1 per cell: a
    sequence holding the diagonal's states scores its length, which only the carry between tile rounds can reach
    (each tile alone sees at most the longer of the two halves).  Also one diagonal inside the first tile (positions
    40..80); no two diagonals of a query overlap, so nothing else on a sequence can add to its score.
    Returns (profiles, sequences, [(query, sequence, score, best single-tile score)])."""
    rng = np.random.default_rng(seed)
    offset = 50
    profs, seqs, cases = [], [], []
    for q, Lq in enumerate(lens):
        p = rng.integers(0, offset - 10, (220, Lq), dtype=np.uint8)
        states = rng.integers(0, 219, Lq).astype(np.uint8)
        spans = [(b - 70 - 13 * k, b + 60 + 11 * k) for k, b in enumerate((512, 1024, 1536)) if b + 60 + 11 * k <= Lq]
        spans.append((40, 80))
        for a, b in spans:
            p[states[a:b], np.arange(a, b)] = offset + 1
            cut = [t for t in (512, 1024, 1536) if a < t < b]
            tile_best = max(cut[0] - a, b - cut[0]) if cut else b - a
            pre = rng.integers(0, 219, int(rng.integers(0, 9)), dtype=np.uint8)
            seqs.append(np.concatenate([pre, states[a:b], rng.integers(0, 219, 5, dtype=np.uint8)]))
            cases.append((q, len(seqs) - 1, b - a, tile_best))
        profs.append(p)
    seqs += [rng.integers(0, 219, L, dtype=np.uint8) for L in (1, 17, 300)]
    return profs, seqs, cases
