"""Seeded inputs at the edges of the over-representation scan (Stats::statRead, src/stats.cpp:270-288; fp_overrep_kernel): evaluated
lengths that make the fifth scan length 0, 1 or equal to one of the first four, reads longer than the evaluated length or filling the
whole row, candidates planted where the scan's loop bound, its skip rule and the kernel's 32-position lane chunks meet, candidate
lists from empty to past the kernel's shared-memory occupancy bitmap, a 64-bit hash collision, and correction-dense pairs whose
pre- and post-filter bases differ.  overrep_case(name, paired, config) returns (params, arrs); every case is deterministic."""
import numpy as np

import edge_inputs as E
import fp_testlib as T
from fastp_b200 import capi

HASH_B = 0x9E3779B97F4A7C15                               # FP_OVERREP_HASH_B of fastp_b200/csrc/fp_device.cuh
M64 = (1 << 64) - 1
# Two distinct 10-byte strings with the same hash (collision_pair() finds them); bytes in [33, 82], so reads holding them fall
# outside A/C/G/T/N and go with the no_filters option set only.
COLLISION_X = b"0!*R!?*!!!"
COLLISION_Y = b"!9!!$!!&PN"
TABLE_BITMAP_BITS = 32768                                 # FP_OVERREP_BM_BITS: a bigger table folds its occupancy bits


def scan_hash(s):
    """The scan's hash of a candidate or window: polynomial in HASH_B over byte + 1, mod 2^64 (0 is stored as 1)."""
    h = 0
    for c in s:
        h = (h * HASH_B + c + 1) & M64
    return h or 1


def table_size(K):
    """Slots of a side's open-addressing table as fp_ctx_create sizes it (1/16 full up to the bitmap size, never above 1/4)."""
    t = 64
    while t < 16 * K and t < TABLE_BITMAP_BITS:
        t <<= 1
    while t < 4 * K:
        t <<= 1
    return t


def collision_pair(n=10, offset=33):
    """How COLLISION_X / COLLISION_Y were found: LLL over the lattice of integer vectors d with sum d_j * B^(n-1-j) = 0 mod 2^64 gives a
    short d (entries <= 49 for n = 10); X_j = offset + max(d_j, 0), Y_j = offset + max(-d_j, 0) then hash alike.  Exact rational
    arithmetic, about 6 s of Python; the tests use the committed constants."""
    from fractions import Fraction
    W = 1 << 40
    b = [[1 if i == j else 0 for j in range(n)] + [W * pow(HASH_B, n - 1 - i, 1 << 64)] for i in range(n)] + [[0] * n + [W << 64]]
    dot = lambda u, v: sum(x * y for x, y in zip(u, v))          # noqa: E731

    def gram_schmidt():
        bs, mu = [], [[Fraction(0)] * len(b) for _ in b]
        for i in range(len(b)):
            v = [Fraction(x) for x in b[i]]
            for j in range(i):
                mu[i][j] = Fraction(dot(b[i], bs[j])) / dot(bs[j], bs[j])
                v = [a - mu[i][j] * c for a, c in zip(v, bs[j])]
            bs.append(v)
        return bs, mu
    bs, mu = gram_schmidt()
    k = 1
    while k < len(b):
        for j in range(k - 1, -1, -1):
            q = round(mu[k][j])
            if q:
                b[k] = [a - q * c for a, c in zip(b[k], b[j])]
                bs, mu = gram_schmidt()
        if dot(bs[k], bs[k]) >= (Fraction(3, 4) - mu[k][k - 1] ** 2) * dot(bs[k - 1], bs[k - 1]):
            k += 1
        else:
            b[k], b[k - 1] = b[k - 1], b[k]
            bs, mu = gram_schmidt()
            k = max(k - 1, 1)
    d = min((r[:n] for r in b if r[-1] == 0 and any(r[:n])), key=lambda r: max(map(abs, r)))
    return bytes(offset + max(v, 0) for v in d), bytes(offset + max(-v, 0) for v in d)


def scan_steps(seq_len):
    return [s for s in (10, 20, 40, 100, min(150, seq_len - 2)) if s > 0]


def _rand(rng, k, alphabet=E.ACGT):
    return rng.choice(alphabet, k).tobytes()


def _rows(n, S, paired, rng, lens, low_ends=False):
    """Random A/C/G/T rows (1 % N) of the given lengths (array or callable(rng, n)), qualities Q25-Q40 with 3 % of Q2-Q16 (most reads
    pass every option set's filters, so the post-filter scan sees them); with low_ends a third of the
    reads get Q2 runs at the front and the tail, so that cut_front / cut_tail / trimming move the post-filter window."""
    _, arrs = capi.host_batch(n, S, paired)
    for sd in ("1", "2")[: 2 if paired else 1]:
        arrs["seq" + sd][:] = rng.choice(E.ACGTN, (n, S), p=[0.2475] * 4 + [0.01])
        q = np.where(rng.random((n, S)) < 0.03, rng.integers(35, 50, (n, S)), rng.integers(58, 74, (n, S))).astype(np.uint8)
        if low_ends:
            j = np.arange(S)[None, :]
            lo = np.where(rng.random(n) < 0.33, rng.integers(0, 12, n), 0)[:, None]
            hi = np.where(rng.random(n) < 0.33, rng.integers(0, 20, n), 0)[:, None]
            ln = np.asarray(lens(rng, n) if callable(lens) else lens, np.int64)[:, None]
            q[(j < lo) | ((j >= ln - hi) & (j < ln))] = 35
            arrs["len" + sd][:] = ln[:, 0]
        else:
            arrs["len" + sd][:] = lens(rng, n) if callable(lens) else lens
        arrs["qual" + sd][:] = q
    return arrs


def _plant(arrs, sd, r, pos, s):
    ln = int(arrs["len" + sd][r])
    if 0 <= pos and pos + len(s) <= ln:
        arrs["seq" + sd][r, pos:pos + len(s)] = np.frombuffer(s, np.uint8)


def _motifs(rng, seq_len, per_step=3):
    """Candidates of every scan length of seq_len: random A/C/G/T strings, the four 1-base strings when the fifth length is 1, one
    string with an N, and strings whose lengths match no scan length."""
    out = []
    for step in scan_steps(seq_len):
        if step == 1:
            out += [b"A", b"C", b"G", b"T"]
        else:
            out += [_rand(rng, step) for _ in range(per_step)]
    out.append(_rand(rng, 4) + b"N" + _rand(rng, 5))
    out += [_rand(rng, 11), _rand(rng, 15), b"ACGTACGTACG"]
    return out


def _plant_edges(arrs, sd, rng, motifs, seq_len):
    """Per read, up to four candidates of the read's own scan lengths: at 0, ending exactly at the read's end (the loop is
    i < len - step, so this one is never counted), one base earlier, and starting at 22-31 (the hit or the position after it lies
    across the first 32-position lane chunk), or at random."""
    steps = [s for s in scan_steps(seq_len) if s > 1]
    by_len = {}
    for m in motifs:
        by_len.setdefault(len(m), []).append(m)
    n = arrs["len" + sd].shape[0]
    for r in range(n):
        ln = int(arrs["len" + sd][r])
        for _ in range(int(rng.integers(0, 5))):
            step = int(rng.choice(steps))
            m = by_len[step][int(rng.integers(0, len(by_len[step])))]
            where = int(rng.integers(0, 5))
            pos = [0, ln - step, ln - step - 1, int(rng.integers(22, 32)), int(rng.integers(0, max(1, ln - step + 1)))][where]
            _plant(arrs, sd, r, pos, m)
        if rng.random() < 0.05:
            _plant(arrs, sd, r, int(rng.integers(0, max(1, ln - 9))), by_len[10][-1] if 10 in by_len else b"")


def _shuffled(rng, cands):
    """Duplicate-free, in a seeded order that is not sorted (the counter index follows the list order)."""
    c = list(dict.fromkeys(cands))
    return [c[i] for i in rng.permutation(len(c))]


def _generic(n, S, paired, rng, seq_lens, lens, low_ends=False):
    arrs = _rows(n, S, paired, rng, lens, low_ends)
    cands = []
    for k, sd in enumerate(("1", "2")[: 2 if paired else 1]):
        m = _motifs(rng, seq_lens[k])
        _plant_edges(arrs, sd, rng, m, seq_lens[k])
        cands.append(_shuffled(rng, m + [_rand(rng, 10) for _ in range(3)]))
    E._zero_padding(arrs)
    return arrs, cands


def _uniform(lo, hi):
    return lambda rng, n: rng.integers(lo, hi + 1, n)


def _lengths_around_steps(S, seq_len):
    """0, 1, step - 1, step, step + 1 of every scan length, S - 1, S, and anything in [0, S]."""
    edges = sorted({0, 1, S - 1, S} | {x for s in scan_steps(seq_len) for x in (s - 1, s, s + 1) if 0 <= x <= S})

    def draw(rng, n):
        v = rng.integers(0, S + 1, n)
        k = min(n, 2 * len(edges))
        v[:k] = np.resize(np.array(edges), k)
        return rng.permutation(v)
    return draw


def _periodic(n, S, paired, rng):
    """Homopolymer, period-2 and period-3 reads: candidates match at every position (or every second / third), so the skip rule
    decides everything.  "AC"*5 and "CA"*5 overlap, and one window matches candidates of two scan lengths ("A"*10 and "A"*20)."""
    units = [b"A", b"AC", b"ACG", b"G", b"CA", b"T"]
    arrs = _rows(n, S, paired, rng, _lengths_around_steps(S, 150))
    for sd in ("1", "2")[: 2 if paired else 1]:
        for r in range(n):
            u = units[r % len(units)]
            ln = int(arrs["len" + sd][r])
            start = int(rng.integers(0, 8)) if r % 3 == 0 else 0          # some reads begin with a few random bases
            body = (u * (S // len(u) + 2))[:max(0, ln - start)]
            arrs["seq" + sd][r, start:start + len(body)] = np.frombuffer(body, np.uint8)
    c = [b"A" * 10, b"A" * 20, b"A" * 40, b"A" * 100, b"A" * 148, b"AC" * 5, b"CA" * 5, b"AC" * 10, b"ACG" * 3 + b"A", b"CGA" * 3 + b"C",
         b"GAC" * 3 + b"G", b"ACG" * 13 + b"A", b"G" * 10, b"G" * 40, b"T" * 20, b"ACGTACGTAC"]
    E._zero_padding(arrs)
    return arrs, [_shuffled(rng, c), _shuffled(rng, c)]


def _wild_bytes(n, S, paired, rng):
    """Bytes outside A/C/G/T/N in reads and candidates (no_filters only): printable 33-126 plus a few above 127."""
    arrs, cands = _generic(n, S, paired, rng, (150, 150), _uniform(100, 150))
    alphabet = np.concatenate([np.arange(33, 127), np.array([128, 200, 255])]).astype(np.uint8)
    out = []
    for k, sd in enumerate(("1", "2")[: 2 if paired else 1]):
        wild = [_rand(rng, step, alphabet) for step in (10, 10, 20, 40) for _ in range(2)]
        for r in range(n):
            ln = int(arrs["len" + sd][r])
            if rng.random() < 0.5:
                arrs["seq" + sd][r, :ln] = rng.choice(alphabet, ln)
            w = wild[int(rng.integers(0, len(wild)))]
            _plant(arrs, sd, r, int(rng.integers(0, ln - len(w) + 1)), w)
        out.append(_shuffled(rng, cands[k] + wild))
    E._zero_padding(arrs)
    return arrs, out


def _collision(n, S, paired, rng, both):
    """Reads holding COLLISION_X and COLLISION_Y (same hash).  both=False: only X is a candidate, so a window holding Y finds X's slot,
    fails the byte compare and counts nothing.  both=True: X and Y are candidates, each counted under its own index (the one inserted
    second sits past the other's slot)."""
    arrs = _rows(n, S, paired, rng, _uniform(60, 150))
    for sd in ("1", "2")[: 2 if paired else 1]:
        for r in range(n):
            ln = int(arrs["len" + sd][r])
            for _ in range(3):
                _plant(arrs, sd, r, int(rng.integers(0, ln - 9)), COLLISION_X if rng.random() < 0.4 else COLLISION_Y)
    E._zero_padding(arrs)
    c1 = [COLLISION_X, COLLISION_Y] if both else [COLLISION_X]
    c2 = [COLLISION_Y, COLLISION_X] if both else [COLLISION_X]
    return arrs, [c1 + [_rand(rng, 10) for _ in range(5)], c2 + [_rand(rng, 20) for _ in range(5)]]


def _many(n, S, paired, rng, K, planted=64):
    """K candidates per side (mostly random 10-mers, some of every scan length); `planted` of them are written into the reads."""
    arrs = _rows(n, S, paired, rng, _uniform(120, 150))
    cands = []
    for sd in ("1", "2")[: 2 if paired else 1]:
        c = set()
        for step, share in ((20, 0.1), (40, 0.05), (100, 0.02), (148, 0.02)):
            c.update(_rand(rng, step) for _ in range(int(K * share)))
        while len(c) < K:
            c.update(rng.choice(E.ACGT, (K - len(c), 10)).view(f"S10")[:, 0].tolist())
        c = _shuffled(rng, sorted(c))[:K]
        for r in range(n):
            ln = int(arrs["len" + sd][r])
            for _ in range(int(rng.integers(0, 4))):
                m = c[int(rng.integers(0, min(planted, K)))]
                _plant(arrs, sd, r, int(rng.integers(0, max(1, ln - len(m)))), m)
        cands.append(c)
    E._zero_padding(arrs)
    return arrs, cands


def dense_correction_candidates(n, rng):
    """Correction-dense pairs (edge_inputs.dense_correction_pairs); for some corrected positions one candidate is the 20 ORIGINAL
    bases around it and one the 20 CORRECTED bases (20, not 10: a random 10-mer turns up by chance in a few hundred reads): the pre-filter scan sees only the first, the post-filter scan only the second.
    Returns (arrs, cands, originals, corrected)."""
    arrs = E.dense_correction_pairs(n, 150, 160, 12, rng)
    p = T.config_params("cfg3_overlap_correction", 1)
    fixed = T.run_cpu("oracle", p, arrs, 160)["arrs"]
    out, orig, corr = [], [], []
    for sd in "12":
        a, b = arrs["seq" + sd], fixed["seq" + sd]
        rows, cols = np.nonzero(a != b)
        o, c = [], []
        for i in rng.permutation(len(rows))[:40]:
            lo = int(np.clip(cols[i] - int(rng.integers(0, 20)), 0, 130))
            w0, w1 = a[rows[i], lo:lo + 20].tobytes(), b[rows[i], lo:lo + 20].tobytes()
            o.append(w0); c.append(w1)
        orig.append(list(dict.fromkeys(o))); corr.append([x for x in dict.fromkeys(c) if x not in o])
        out.append(_shuffled(rng, orig[-1] + corr[-1]))
    return arrs, out, orig, corr


# name -> (paired only?, option sets it is restricted to or None)
CASES = {
    "evallen_2": (False, None), "evallen_3": (False, None), "evallen_12_22": (False, None), "evallen_42_102": (False, None),
    "evallen_below_reads": (False, None), "evallen_above_stride": (False, None),
    "full_stride": (False, None), "full_stride_304": (False, None), "full_stride_512": (False, None),
    "read_lengths": (False, None), "trimmed_windows": (False, None), "skip_rule": (False, None), "bytes_n": (False, None),
    "bytes_wild": (False, ("no_filters",)), "collision_x_only": (False, ("no_filters",)), "collision_both": (False, ("no_filters",)),
    "k0_side1": (False, None), "k0_side2": (True, None), "k0_both": (False, None), "k1": (False, None),
    "k2048": (False, None), "k2049": (False, None), "k8192": (False, None), "k8193": (False, None), "k20000": (False, None),
    "dense_correction": (True, None),
}
CONFIGS = ["all_cuts", "cfg3_overlap_correction", "cfg4_full", "no_filters"]


def case_ids(paired, configs=CONFIGS):
    """(case, config) pairs valid for SE (paired=0) or PE (paired=1)."""
    return [(c, cfg) for c, (pe_only, only) in CASES.items() for cfg in configs if (paired or not pe_only) and (only is None or cfg in only)]


def overrep_inputs(name, paired, n=None, seed=0):
    """(arrs, [candidates1, candidates2], (seq_len1, seq_len2)) of one case."""
    rng = np.random.default_rng(hash_name(name) + 1000 * seed + paired)
    pe_S = 256
    if name.startswith("evallen_"):
        sl = {"evallen_2": (2, 3), "evallen_3": (3, 2), "evallen_12_22": (12, 22), "evallen_42_102": (42, 102),
              "evallen_below_reads": (60, 100), "evallen_above_stride": (300, 280)}[name]
        S = 256 if name == "evallen_above_stride" else 160
        arrs, c = _generic(n or 500, S, paired, rng, sl, _lengths_around_steps(S, min(sl)))
        return arrs, c, sl
    if name.startswith("full_stride"):
        S = pe_S if paired or name == "full_stride" else int(name.rsplit("_", 1)[1])
        arrs, c = _generic(n or 400, S, paired, rng, (S, S - 6), lambda rng, k: np.full(k, S))
        return arrs, c, (S, S - 6)
    if name == "read_lengths":
        arrs, c = _generic(n or 600, 160, paired, rng, (150, 150), _lengths_around_steps(160, 150))
        return arrs, c, (150, 150)
    if name == "trimmed_windows":
        arrs, c = _generic(n or 600, 160, paired, rng, (150, 140), _uniform(0, 160), low_ends=True)
        return arrs, c, (150, 140)
    if name == "skip_rule":
        arrs, c = _periodic(n or 600, 160, paired, rng)
        return arrs, c, (150, 150)
    if name == "bytes_n":
        arrs, c = _generic(n or 500, 160, paired, rng, (150, 150), _uniform(60, 160))
        for k, sd in enumerate(("1", "2")[: 2 if paired else 1]):
            nn = [b"N" * 10, b"ACGTNNACGT", b"N" + _rand(rng, 19)]
            for r in range(0, arrs["seq1"].shape[0], 3):
                _plant(arrs, sd, r, int(rng.integers(0, 50)), nn[r % 3])
            c[k] = _shuffled(rng, c[k] + nn)
        return arrs, c, (150, 150)
    if name == "bytes_wild":
        arrs, c = _wild_bytes(n or 500, 160, paired, rng)
        return arrs, c, (150, 150)
    if name.startswith("collision_"):
        arrs, c = _collision(n or 400, 160, paired, rng, name == "collision_both")
        return arrs, c, (150, 150)
    if name.startswith("k0_") or name == "k1":
        arrs, c = _generic(n or 500, 160, paired, rng, (150, 150), _uniform(100, 160))
        if name == "k1":
            c = [[x for x in cc if len(x) == 10][:1] for cc in c]
            for sd, cc in zip("12", c):
                for r in range(0, arrs["seq1"].shape[0], 2):
                    _plant(arrs, sd, r, int(rng.integers(0, 90)), cc[0])
        else:
            empty = {"k0_side1": (0,), "k0_side2": (1,), "k0_both": (0, 1)}[name]
            c = [[] if k in empty else cc for k, cc in enumerate(c)]
        return arrs, c, (150, 150)
    if name.startswith("k"):
        arrs, c = _many(n or 300, 160, paired, rng, int(name[1:]))
        return arrs, c, (150, 150)
    if name == "dense_correction":
        arrs, c, _, _ = dense_correction_candidates(n or 400, rng)
        return arrs, c, (150, 150)
    raise KeyError(name)


def hash_name(name):
    return sum((i + 1) * ord(ch) for i, ch in enumerate(name))


def with_overrep(p, cands, seq_lens, sampling, paired):
    kw = dict(overrep_enabled=1, overrep_sampling=sampling, seq_len1=seq_lens[0], seq_len2=seq_lens[1], overrep_seqs1=cands[0])
    if paired:
        kw["overrep_seqs2"] = cands[1]
    capi.set_params(p, **kw)
    return p


def overrep_case(name, paired, config="no_filters", sampling=1, n=None, seed=0):
    """(params, arrs) of one case under one option set; cycles = the row stride."""
    arrs, cands, sl = overrep_inputs(name, paired, n, seed)
    p = T.config_params(config, paired)
    return with_overrep(p, cands, sl, sampling, paired), arrs
