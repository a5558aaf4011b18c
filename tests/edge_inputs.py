"""Seeded generators of inputs at the edges of the parity domain (DESIGN §3): every quality byte in [33, 126], read lengths
up to the full row stride, pairs dense enough in corrections to overflow the per-tile and per-chunk correction lists, and
reads whose 3' end trims once per fasta adapter.  They write into capi.host_batch arrays and keep every padding byte zero."""
import numpy as np

from fastp_b200 import capi

ACGT = np.frombuffer(b"ACGT", np.uint8)
ACGTN = np.frombuffer(b"ACGTN", np.uint8)
LENGTH_EDGES = (0, 1, 31, 32, 33, 63, 64, 65)          # word and plane boundaries; S - 1 and S are added per stride


def _sides(arrs):
    return ("1", "2") if "seq2" in arrs else ("1",)


def _zero_padding(arrs):
    S = arrs["seq1"].shape[1]
    for sd in _sides(arrs):
        pad = np.arange(S)[None, :] >= arrs["len" + sd].astype(np.int64)[:, None]
        arrs["seq" + sd][pad] = 0
        arrs["qual" + sd][pad] = 0


def quality_thresholds(p):
    """Quality bytes on both sides of every threshold option set `p` uses: qualified_qual, the cut_* window qualities,
    Q20 / Q30 (52 / 53, 62 / 63) and the base correction's BAD / GOOD cut-offs (47 / 48, 62 / 63)."""
    t = {p.qualified_qual - 1, p.qualified_qual, 52, 53, 62, 63, 47, 48}
    for q in (p.cut_front_quality, p.cut_tail_quality, p.cut_right_quality):
        t.update((33 + q - 1, 33 + q, 33 + q + 1))
    return np.array(sorted(x for x in t if 33 <= x <= 126), np.uint8)


def quality_extremes(arrs, rng, p):
    """Rewrite the qualities of each read in one of these modes: unchanged (a quarter of the reads), uniform over [33, 126],
    all 33 (Q0), all 126 (Q93), or drawn from quality_thresholds(p).  Bases and lengths stay as they are."""
    thr = quality_thresholds(p)
    S = arrs["seq1"].shape[1]
    for sd in _sides(arrs):
        q = arrs["qual" + sd]
        n = q.shape[0]
        mode = rng.choice(5, n, p=[0.25, 0.25, 0.1, 0.1, 0.3])
        q[mode == 1] = rng.integers(33, 127, (int((mode == 1).sum()), S), dtype=np.uint8)
        q[mode == 2] = 33
        q[mode == 3] = 126
        q[mode == 4] = rng.choice(thr, (int((mode == 4).sum()), S))
    _zero_padding(arrs)
    return arrs


def ragged_lengths(arrs, rng, S):
    """Draw the lengths of read 1 and read 2 independently from [0, S] (S <= the row stride): with at least S + 1 reads every
    value appears, and 0, 1, 31-33, 63-65, S - 1 and S make up about a third of the reads.  Bases a read gains are random
    A/C/G/T (1 % N) with qualities in [35, 73]."""
    stride = arrs["seq1"].shape[1]
    assert S <= stride
    edges = np.array(sorted({x for x in LENGTH_EDGES if x <= S} | {S - 1, S}), np.int64)
    for sd in _sides(arrs):
        seq, q, ln = arrs["seq" + sd], arrs["qual" + sd], arrs["len" + sd]
        n = ln.shape[0]
        old = ln.astype(np.int64)
        new = rng.integers(0, S + 1, n)
        order = rng.permutation(n)
        k = min(n, S + 1)
        new[order[:k]] = rng.permutation(S + 1)[:k]
        m = min(n - k, n // 3)
        new[order[k:k + m]] = rng.choice(edges, m)
        grow = np.arange(stride)[None, :] >= old[:, None]
        bases = rng.choice(ACGTN, (n, stride), p=[0.2475] * 4 + [0.01])
        seq[grow] = bases[grow]
        q[grow] = rng.integers(35, 74, (n, stride), dtype=np.uint8)[grow]
        ln[:] = new
    _zero_padding(arrs)
    return arrs


def edge_batch(n, S, paired, seed, p, read_len=None, max_len=None):
    """Synthetic rows (profile 1) with ragged_lengths up to max_len (default: the stride S) and then quality_extremes applied:
    the quality x length grid input."""
    import fp_testlib as T
    _, arrs = T.synth_host(n, S, paired, seed * 1000, seed, 1, read_len or min(150, S))
    rng = np.random.default_rng(seed)
    ragged_lengths(arrs, rng, max_len or S)
    quality_extremes(arrs, rng, p)
    return arrs


def dense_correction_pairs(n, L, S, k, rng):
    """Pairs that overlap over their whole insert (L - 20 to L bases) with k planted mismatches in the overlap: at each one,
    one side holds a changed base at Q2-Q14 and the other side the true base at Q30-Q93 (quality bytes 63-126); every other
    base is Q37.  With --correction most mismatches are corrected (about 9.5 per pair at overlap_diff_limit 5 and k = 12),
    far more than FP_CORR_CAP per tile and more than two per pair per host chunk."""
    _, arrs = capi.host_batch(n, S, 1)
    for lo in range(0, n, 1 << 15):                          # blocks keep the temporaries small at a few 100 000 pairs
        _dense_block(arrs, lo, min(n, lo + (1 << 15)), L, k, rng)
    arrs["len1"][:] = L
    arrs["len2"][:] = L
    return arrs


def _dense_block(arrs, lo, hi, L, k, rng):
    n = hi - lo
    rows = np.arange(n)[:, None]
    j = np.arange(L)[None, :]
    ins = rng.integers(L - 20, L + 1, n)
    r1 = rng.integers(0, 4, (n, L), dtype=np.uint8)          # codes A0 C1 G2 T3: 3 - x is the complement
    src = ins[:, None] - 1 - j                               # read 2 position j holds the complement of fragment position ins-1-j
    r2 = np.where(src >= 0, 3 - r1[rows, np.maximum(src, 0)], rng.integers(0, 4, (n, L), dtype=np.uint8)).astype(np.uint8)
    q1 = np.full((n, L), 33 + 37, np.uint8)
    q2 = np.full((n, L), 33 + 37, np.uint8)
    key = np.where((j >= 2) & (j < ins[:, None] - 2), rng.random((n, L), dtype=np.float32), np.float32(np.inf))
    f = np.argsort(key, axis=1)[:, :k]                       # k distinct fragment positions in [2, ins - 2)
    p2 = ins[:, None] - 1 - f
    bad = rng.integers(33 + 2, 33 + 15, (n, k)).astype(np.uint8)
    good = rng.integers(33 + 30, 33 + 94, (n, k)).astype(np.uint8)
    on1 = rng.random((n, k)) < 0.5                           # which side carries the error
    rr = np.broadcast_to(rows, (n, k))
    a, b = (rr[on1], f[on1]), (rr[on1], p2[on1])
    r1[a] = (r1[a] + 1) % 4
    q1[a] = bad[on1]
    q2[b] = good[on1]
    a, b = (rr[~on1], p2[~on1]), (rr[~on1], f[~on1])
    r2[a] = (r2[a] + 1) % 4
    q2[a] = bad[~on1]
    q1[b] = good[~on1]
    arrs["seq1"][lo:hi, :L] = ACGT[r1]
    arrs["seq2"][lo:hi, :L] = ACGT[r2]
    arrs["qual1"][lo:hi, :L] = q1
    arrs["qual2"][lo:hi, :L] = q2


def adapter_concatemers(n, S, adapters, rng, paired=1):
    """Reads made of a random insert followed by the adapters in REVERSE list order, cut to S bases: trimByMultiSequences then
    trims the last adapter with the first list entry, the one before it with the second and so on, one addAdapterTrimmed call
    per adapter.  The two reads of a pair are independent (no overlap), so a pair gives up to 2 + 2 * len(adapters) events."""
    _, arrs = capi.host_batch(n, S, paired)
    tail = np.frombuffer("".join(reversed(adapters)).encode(), np.uint8)
    for sd in ("1", "2")[: 2 if paired else 1]:
        ins = rng.integers(max(0, S - len(tail) - 40), max(1, S - len(tail)) + 1, n)
        seq = rng.choice(ACGT, (n, S))
        pos = np.arange(S)[None, :] - ins[:, None]
        body = pos >= 0
        seq[body] = tail[np.minimum(pos[body], len(tail) - 1)]
        ln = np.minimum(ins + len(tail), S)
        arrs["seq" + sd][:] = seq
        arrs["qual" + sd][:] = rng.integers(33 + 30, 33 + 41, (n, S), dtype=np.uint8)
        arrs["len" + sd][:] = ln
    _zero_padding(arrs)
    return arrs
