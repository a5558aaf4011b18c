"""Option sets at the ends of every option's accepted range, and inputs that sit exactly on each filter's threshold (DESIGN §3).

option_edge_sets(paired) lists named option sets.  Each starts from a base config and moves one option, or one coupled group of
options, to an edge value.  A set's name begins with the kernel branch it targets (cut_right.scalar, polyg.plane_off,
overlap.filter_wide, isize.global, ...), so a failure names the branch.  Values that depend on the input are written as L (the
read length of the edge batch, min(150, S)) and S (the row stride) and resolved per stride by edge_params().

threshold_batch(p, S, paired, seed) builds reads that put one predicate of option set p exactly on its limit (label at = 0) and
the next read one past it (at = 1), with every other predicate far from its own limit where p allows it: the passFilter counts
(low-quality bases, N bases, the average quality, adjacent differences), the first trimAndCut window of cut_front / cut_tail /
cut_right, the overlap mismatch limit, and polyG / polyX tails of minLen - 1 and minLen.  boundary_outcomes() reads the oracle's
records back and reports, per predicate, how many reads on each side of the limit came out as that side should.  Padding bytes are
zero, as in tests/edge_inputs.py."""
import numpy as np

from fastp_b200 import capi

import fp_testlib as T

ACGT = b"ACGT"
FP_PASS_FILTER, FP_FAIL_N_BASE, FP_FAIL_QUALITY, FP_FAIL_COMPLEXITY = 0, 12, 20, 24

CUT_WINDOWS = ("1", "2", "3", "4", "5", "8", "9", "31", "32", "33", "L-1", "L", "L+1", "1000")
POLY_MIN_LENS = ("0", "1", "2", "5", "6", "8", "9", "10", "11", "31", "32", "33", "64", "L", "L+1", "S+1")
OV_REQUIRES = ("0", "1", "2", "31", "32", "33", "50", "L-1", "L", "L+1")
OV_DIFF_LIMITS = ("0", "31", "32", "33", "51", "1000")
OV_DIFF_PERCENTS = (0, 1, 100)
TRIMS = ("L-1", "L", "L+1", "S")
ISIZE_MAXES = (0, 1, 1023, 1024, 1025, 4096)      # FP_MAX_ISIZE_SMEM = 1025: from there on every insert size goes to the global bins

# the passFilter sets run on this base: no trimming of any kind, so threshold reads reach passFilter as they were built
FILTER_BASE = dict(adapter_enabled=0, length_required=1)


def _tok(v):
    return str(v).replace("+", "p").replace("-", "m")


def _cut_right_tag(w):
    # windows <= 8 on clean rows walk plane 4; w == 4 on other rows sums one dp4a field; everything else is the scalar rolling sum
    if w in ("4",):
        return "cut_right.plane4_dp4a"
    if w in ("1", "2", "3", "5", "8"):
        return "cut_right.plane4"
    return "cut_right.scalar"


def _poly_tags(m):
    try:
        v = int(m)
    except ValueError:
        v = 1000                                   # L, L+1, S+1: always above 32 here
    g = "polyg.plane_off" if v > 32 or v < 1 else "polyg.plane"
    x = "polyx.plane" if v >= 10 else "polyx.scan"
    return g + "+" + x


def _ov_tag(req, dl, pct):
    tags = []
    r = {"L-1": 99, "L": 100, "L+1": 101}.get(req, None)
    r = int(req) if r is None else r
    tags.append("filter_req_le1" if r <= 1 else "filter_narrow" if r < 32 else "filter_wide")
    if dl is not None and pct == 100 and dl not in ("0", "31"):
        tags.append("thr_gt32")                  # lut[ol] + 1 > 32 for long overlaps: the filter passes every candidate
    return "overlap." + "+".join(tags)


def option_edge_sets(paired):
    """name -> keyword set (values may be 'L', 'S' expressions).  Merging-mode sets are the ones whose name starts with 'merge'."""
    sets = {}

    def add(name, **kw):
        assert name not in sets, name
        sets[name] = kw

    for w in CUT_WINDOWS:
        for q in (1, 30):
            add(f"cut_front_tail.w{_tok(w)}_q{q}", cut_front=1, cut_tail=1, cut_front_window=w, cut_tail_window=w,
                cut_front_quality=q, cut_tail_quality=q)
            add(f"{_cut_right_tag(w)}.w{_tok(w)}_q{q}", cut_right=1, cut_right_window=w, cut_right_quality=q)
    for m in POLY_MIN_LENS:
        add(f"{_poly_tags(m)}.min{_tok(m)}", polyg_enabled=1, polyx_enabled=1, polyg_min_len=m, polyx_min_len=m)
    for m in ("10", "30", "33"):                  # polyG alone: its boundary reads are not cut by polyX
        add(f"{_poly_tags(m).split('+')[0]}.only_min{m}", polyg_enabled=1, polyg_min_len=m)
    for q in (0, 1, 93):
        add(f"filter.qualified_q{q}", **FILTER_BASE, qualified_qual=33 + q)
    for pct in (0, 1, 50, 99, 100):
        add(f"filter.unqualified_pct{pct}", **FILTER_BASE, unqualified_percent_limit=pct)
    for a in (1, 20, 93):
        add(f"filter.avg_qual{a}", **FILTER_BASE, avg_qual_req=a, qualified_qual=33)
    for n in (0, 50):
        add(f"filter.n_base_limit{n}", **FILTER_BASE, n_base_limit=n)
    for c in (0, 1, 33, 50, 99, 100):
        add(f"filter.complexity{c}", **FILTER_BASE, complexity_filter_enabled=1, complexity_threshold=c / 100.0)
    for r in ("0", "1", "S", "S+1"):
        add(f"filter.length_required{_tok(r)}", **dict(FILTER_BASE, length_required=r))
    for m in ("1", "S-1", "S"):
        add(f"filter.length_limit{_tok(m)}", **FILTER_BASE, length_limit=m)
    for t in TRIMS:
        add(f"trim.t{_tok(t)}", trim_front1=t, trim_tail1=t if not paired else 0, trim_tail2=t if paired else 0)
        add(f"trim_cut.t{_tok(t)}", trim_front1=t, trim_tail2=t if paired else 0, cut_front=1, cut_right=1)
    for m in ("1", "2", "S"):
        add(f"trim.max_len{_tok(m)}", max_len1=m, max_len2=m if paired else 0)
    for d in ("0", "L", "S"):
        add(f"adapter.dimer_max_len{_tok(d)}", dimer_max_len=d, adapter_seq_r1=T.TRUSEQ_R1)
    # thread0_semantics 0 (the counters of a worker other than the first) on a few of the above
    add("tid1.cut_right.plane4_dp4a.w4_q30", thread0_semantics=0, cut_right=1, cut_right_window=4, cut_right_quality=30)
    add("tid1.polyg.plane_off+polyx.plane.min33", thread0_semantics=0, polyg_enabled=1, polyx_enabled=1, polyg_min_len=33, polyx_min_len=33)
    add("tid1.filter.unqualified_pct0", thread0_semantics=0, **FILTER_BASE, unqualified_percent_limit=0)
    if paired:
        for r in OV_REQUIRES:
            add(f"{_ov_tag(r, None, None)}.req{_tok(r)}", overlap_require=r, correction_enabled=1)
            add(f"{_ov_tag(r, None, None)}.req{_tok(r)}_plain", overlap_require=r, adapter_enabled=0)
            if r not in ("0", "1"):              # the one-gap pass needs overlap_require >= 2 (fp_ctx_create refuses less)
                add(f"{_ov_tag(r, None, None)}.req{_tok(r)}_gap", overlap_require=r, correction_enabled=1, allow_gap_overlap_trimming=1)
        for dl in OV_DIFF_LIMITS:
            for pct in OV_DIFF_PERCENTS:
                add(f"{_ov_tag('30', dl, pct)}.diff{dl}_pct{pct}", overlap_diff_limit=dl, overlap_diff_percent_limit=pct, correction_enabled=1,
                    allow_gap_overlap_trimming=int(dl in ("0", "33", "1000")))
        add("overlap.filter_req_le1+thr_gt32.req1_diff1000_pct100", overlap_require=1, overlap_diff_limit=1000, overlap_diff_percent_limit=100,
            correction_enabled=1)
        add("overlap.threshold", adapter_enabled=0, correction_enabled=1)
        for im in ISIZE_MAXES:
            add(f"isize.{'global' if im >= 1025 else 'smem'}.max{im}", insert_size_max=im)
        add("tid1.overlap.filter_wide.req33", thread0_semantics=0, overlap_require=33, correction_enabled=1)
        # merging mode (forces --correction): the passFilter and overlap sets again, merged reads up to 2 * S long
        base = [k for k in sets if k.startswith(("filter.", "overlap."))]
        for i, k in enumerate(base):
            kw = dict(sets[k], merge_enabled=1, correction_enabled=1, merge_include_unmerged=i % 2)
            add(("mergeu." if i % 2 else "merge.") + k, **kw)
    return sets


def resolve(kw, S, L):
    env = {"S": S, "L": L}
    return {k: (eval(v, {}, env) if isinstance(v, str) and k != "adapter_seq_r1" else v) for k, v in kw.items()}   # noqa: S307


def read_len(S):
    return min(150, S)


def edge_params(name, paired, S, lib=None):
    kw = resolve(option_edge_sets(paired)[name], S, read_len(S))
    return capi.default_params(paired, lib=lib or T.oracle(), **kw)


def cycles_for(name, S):
    return 2 * S if name.startswith("merge") else S


# ---------------- threshold reads ----------------
KINDS = ("fill", "lowq", "nbase", "avgq", "complexity", "cut_front", "cut_tail", "cut_right", "overlap", "polyg", "polyx")
K = {k: i for i, k in enumerate(KINDS)}


class _Side:
    def __init__(self):
        self.rows = []                            # (seq bytes, qual bytes, kind, at, want)

    def add(self, seq, qual, kind, at, want=0):
        assert len(seq) == len(qual)
        self.rows.append((bytes(seq), bytes(qual), K[kind], at, want))


def _rand_bases(rng, n, avoid_end=None):
    s = bytearray(rng.choice(np.frombuffer(ACGT, np.uint8), n).tobytes())
    if avoid_end is not None and n:
        while s[-1] == avoid_end:
            s[-1] = ACGT[int(rng.integers(0, 4))]
    return s


def _hq(p):
    """A quality byte above every per-base threshold of p (qualified_qual and the three cut qualities)."""
    return min(126, max(p.qualified_qual, 33 + max(p.cut_front_quality, p.cut_tail_quality, p.cut_right_quality) + 1, 33 + 40))


def _sample_lens(rng, lo, S, k=12):
    if lo > S:
        return []
    base = {lo, lo + 1, 31, 32, 33, 63, 64, 65, S - 1, S}
    base |= set(int(x) for x in rng.integers(lo, S + 1, k))
    return sorted(x for x in base if lo <= x <= S)


def _pass_filter_reads(p, S, rng, out):
    hq = _hq(p)
    lq = p.qualified_qual - 1
    pct = p.unqualified_percent_limit
    if lq >= 33:                                  # lowQualNum > pct * rlen / 100.0: floor(pct * rlen / 100) passes, one more fails
        for rlen in range(1, S + 1):
            k = pct * rlen // 100
            for at in (0, 1):
                m = k + at
                if m > rlen:
                    continue
                q = bytearray([hq] * rlen)
                for i in rng.choice(rlen, m, replace=False):
                    q[i] = lq
                out.add(_rand_bases(rng, rlen), q, "lowq", at)
    nl = p.n_base_limit                           # nBaseNum > nBaseLimit
    for rlen in _sample_lens(rng, max(nl + 1, 1), S):
        for at in (0, 1):
            m = nl + at
            if m > rlen:
                continue
            s = _rand_bases(rng, rlen)
            for i in rng.choice(rlen, m, replace=False):
                s[i] = ord("N")
            out.add(s, [hq] * rlen, "nbase", at)
    a = p.avg_qual_req                            # totalQual / rlen < avgQualReq (integer division)
    if a > 0:
        vmin = max(0, p.qualified_qual - 33)
        for rlen in _sample_lens(rng, 1, S):
            for at in (0, 1):
                tot = a * rlen + (int(rng.integers(0, rlen)) if a < 93 else 0) if at == 0 else a * rlen - 1
                if tot < 0 or tot > 93 * rlen:
                    continue
                base, extra = divmod(tot, rlen)
                v = np.full(rlen, base, np.int64)
                v[rng.choice(rlen, extra, replace=False)] += 1
                if v.min() < vmin and at == 0:
                    continue
                out.add(_rand_bases(rng, rlen), (v + 33).astype(np.uint8).tobytes(), "avgq", at)
    if p.complexity_filter_enabled:               # (double)diff / (double)(rlen - 1) >= threshold
        thr = p.complexity_threshold
        lens = range(2, S + 1) if S <= 160 else _sample_lens(rng, 2, S, 48)
        for rlen in lens:
            dmin = next((k for k in range(rlen) if k / (rlen - 1) >= thr), None)
            if dmin is None:
                continue
            for at in (0, 1):
                d = dmin - at
                if d < 0:
                    continue
                trans = set(int(x) for x in rng.choice(np.arange(1, rlen), d, replace=False))
                s = bytearray(rlen)
                s[0] = ACGT[int(rng.integers(0, 4))]
                for i in range(1, rlen):
                    s[i] = s[i - 1] if i not in trans else ACGT[(ACGT.index(s[i - 1]) + int(rng.integers(1, 4))) % 4]
                out.add(s, [hq] * rlen, "complexity", at)


POSITIONS = (0, 1, 30, 31, 32, 33, 62, 63, 64, 65, 95, 96, 127, 128)


def _cut_reads(p, S, rng, out):
    hq = _hq(p)
    for kind, on, w, Q in (("cut_front", p.cut_front, p.cut_front_window, p.cut_front_quality),
                           ("cut_tail", p.cut_tail and not p.cut_right, p.cut_tail_window, p.cut_tail_quality),
                           ("cut_right", p.cut_right, p.cut_right_window, p.cut_right_quality)):
        if not on:
            continue
        thr_q = 33 + Q
        if hq <= thr_q or thr_q - 1 < 33:
            continue
        for rlen in sorted({S, max(1, S - 7)}):
            for pos in sorted(set(POSITIONS) | {max(0, rlen - w - 2)}):
                if kind == "cut_right":
                    # every window sums to exactly w * (33 + Q) (not < the threshold: no cut); one base one lower makes the first window
                    # that holds it the cut, and the cut then ends at that base
                    if pos == 0 or pos >= rlen - 1:
                        continue
                    for at in (0, 1):
                        q = bytearray([thr_q] * rlen)
                        if at:
                            q[pos] = thr_q - 1
                        s = _rand_bases(rng, rlen)
                        want = rlen if not at else pos
                        out.add(s, q, kind, at, want)
                        s2 = bytearray(s)                 # the same read with one byte outside A/C/G/T/N: the row takes the byte paths
                        s2[-1] = ord("R")
                        out.add(s2, q, kind, 2, want)
                    continue
                if pos + w + 1 >= rlen:
                    continue
                for at in (0, 1):
                    for nrun in (0, 3):
                        # bases before the window at Q0 (every earlier window sums below), the window exactly at w * (33 + Q) or one
                        # below, bases after it high; nrun N bases where the cut lands (the reference skips them)
                        q = bytearray([33] * pos + [thr_q] * w + [hq] * (rlen - pos - w))
                        if at:
                            q[pos + w - 1] = thr_q - 1
                        s = _rand_bases(rng, rlen)
                        cut = pos + w - 1 if pos > 0 else 0
                        for i in range(cut, min(rlen, cut + nrun)):
                            s[i] = ord("N")
                        want = cut + (nrun if nrun and cut + nrun < rlen else 0)
                        if kind == "cut_tail":              # the mirror image: the window counted from the 3' end
                            q, s = q[::-1], s[::-1]
                            want = rlen - want
                        out.add(s, q, kind, 2 if at and nrun else at, want)     # one past with N bases: the skip lands on the same base


def _poly_reads(p, S, rng, out):
    hq = _hq(p)
    for kind, on, m in (("polyg", p.polyg_enabled, p.polyg_min_len), ("polyx", p.polyx_enabled, p.polyx_min_len)):
        if not on:
            continue
        if kind == "polyg" and 1 <= m <= 39 and m + 1 < S:
            # trimPolyG trims iff its scan ends at i >= minLen (i counts from the 3' end).  k = m // 8 + 1 non-G bases, k - 1 of them at
            # i = 0 .. k-2 and the last at i = m - 1, end it there (no trim, at 1); the last at i = m ends it one base later (trim, at 0)
            k = m // 8 + 1
            for at, last in ((0, m), (1, m - 1)):
                if k > 5 or k - 2 >= last or (at == 0 and (m + 1) % 8 == 0):
                    continue
                for rlen in (S, int(rng.integers(m + 2, S + 1))):
                    s = _rand_bases(rng, rlen)
                    for i in range(last):
                        s[rlen - 1 - i] = ord("G")
                    for i in list(range(k - 1)) + [last]:
                        s[rlen - 1 - i] = ACGT[int(rng.integers(0, 3))]          # A, C or G -> A, C, T below
                        if s[rlen - 1 - i] == ord("G"):
                            s[rlen - 1 - i] = ord("T")
                    out.add(s, [hq] * rlen, kind, at, rlen)
        for t in (m - 1, m, m + 1):
            if t < 1 or t > S - 1:
                continue
            for variant in range(3):
                rlen = int(rng.integers(t + 1, S + 1)) if variant else S
                b = ord("G") if kind == "polyg" else ACGT[int(rng.integers(0, 4))]
                s = _rand_bases(rng, rlen - t, avoid_end=b) + bytearray([b] * t)
                if variant == 1:                        # mismatches at the 8m - 2 break points, counted from the 3' end
                    for i in (6, 14, 22):
                        if i < t:
                            s[rlen - 1 - i] = ACGT[(ACGT.index(b) + 1) % 4]
                if variant == 2:
                    for i in (7, 15):
                        if i < t:
                            s[rlen - 1 - i] = ord("N") if kind == "polyx" else ord("T")
                out.add(s, [hq] * rlen, kind, 2, rlen)


def _rc(s):
    return bytes(bytearray(b"TGCAN"[b"ACGTN".index(c)] for c in reversed(s)))


def ov_limit(p, ol):
    return min(p.overlap_diff_limit, int(ol * (p.overlap_diff_percent_limit / 100.0)))       # overlapanalysis.cpp:51


def _overlap_pairs(p, S, rng, o1, o2):
    """Pairs of equal length n whose candidate at offset +o or -o (ol = n - o) holds exactly lut[ol] (at 0) or lut[ol] + 1 (at 1)
    mismatches in its first min(ol, 50) compared bases, and pairs with mismatches only past base 50 (at 2)."""
    hq = _hq(p)
    req = p.overlap_require
    ols = sorted({req + 1, req + 2, 31, 32, 33, 49, 50, 51, 52, 63, 64, 65, S - 1, S} | set(int(x) for x in rng.integers(1, S + 1, 6)))
    for n in sorted({S, max(1, S - 5)}):
        for ol in ols:
            if ol < max(req + 1, 1) or ol > n:
                continue
            o = n - ol
            pp = min(ol, 50)
            for sign in (1, -1):
                if sign < 0 and o == 0:
                    continue
                for at in (0, 1, 2):
                    mm = ov_limit(p, ol) + at if at < 2 else 0
                    if mm > pp or (at == 2 and ol <= 50):
                        continue
                    X = _rand_bases(rng, n)               # X = rc(read 2)
                    r1 = _rand_bases(rng, n)
                    if sign > 0:                          # r1[o + k] vs X[k]
                        r1[o:o + ol] = X[:ol]
                        base1 = o
                    else:                                 # r1[k] vs X[o + k]
                        r1[:ol] = X[o:o + ol]
                        base1 = 0
                    ks = rng.choice(pp, mm, replace=False) if at < 2 else 50 + rng.choice(ol - 50, int(rng.integers(1, min(10, ol - 50) + 1)), replace=False)
                    for k in ks:
                        i = base1 + int(k)
                        r1[i] = ACGT[(ACGT.index(r1[i]) + int(rng.integers(1, 4))) % 4]
                    want = sign * o
                    o1.add(r1, [hq] * n, "overlap", at, want)
                    o2.add(_rc(X), [hq] * n, "overlap", at, want)


def threshold_batch(p, S, paired, seed):
    """(arrs, labels): rows at stride S that sit on the thresholds of option set p; labels[side] is a structured array
    (kind, at, want) per read.  Pairs of the non-overlap kinds hold two unrelated threshold reads."""
    rng = np.random.default_rng(seed)
    sides = [_Side(), _Side()] if paired else [_Side()]
    for sd in sides:
        _pass_filter_reads(p, S, rng, sd)
        _cut_reads(p, S, rng, sd)
        _poly_reads(p, S, rng, sd)
    if paired:                                    # the two sides' single-read lists, side 2 shuffled against side 1
        a, b = sides
        b.rows = [b.rows[i] for i in rng.permutation(len(b.rows))]
        n = max(len(a.rows), len(b.rows))
        for sd in sides:
            while len(sd.rows) < n:
                rlen = int(rng.integers(0, S + 1))
                sd.add(_rand_bases(rng, rlen), [_hq(p)] * rlen, "fill", 2)
        _overlap_pairs(p, S, rng, a, b)
    n = len(sides[0].rows)
    order = rng.permutation(n)
    _, arrs = capi.host_batch(n, S, 1 if paired else 0)
    lab_dtype = np.dtype([("kind", "i1"), ("at", "i1"), ("want", "<i4")])
    labels = {}
    for k, sd in enumerate(sides):
        tag = str(k + 1)
        lab = np.zeros(n, lab_dtype)
        for r, i in enumerate(order):
            s, q, kind, at, want = sd.rows[i]
            arrs["seq" + tag][r, :len(s)] = np.frombuffer(s, np.uint8)
            arrs["qual" + tag][r, :len(q)] = np.frombuffer(q, np.uint8)
            arrs["len" + tag][r] = len(s)
            lab[r] = (kind, at, want)
        labels[tag] = lab
    return arrs, labels


def boundary_outcomes(labels, res, paired):
    """kind -> [reads on the limit that came out as 'on the limit', reads on the limit, reads one past that came out as 'one past',
    reads one past], from the records of `res` (fp_testlib.run_cpu or fp_gpu.run_gpu)."""
    out = {}
    for tag in ("1", "2")[: 2 if paired else 1]:
        lab, rec = labels[tag], res["out" + tag]
        v, front, ln = rec["verdict"].astype(int), rec["front"].astype(int), rec["len"].astype(int)
        ov = res["ov"] if paired else None
        for kind in KINDS[1:]:
            for at in (0, 1):
                sel = (lab["kind"] == K[kind]) & (lab["at"] == at)
                if not sel.any():
                    continue
                want = lab["want"][sel]
                if kind in ("lowq", "avgq", "nbase", "complexity"):
                    fail = {"lowq": FP_FAIL_QUALITY, "avgq": FP_FAIL_QUALITY, "nbase": FP_FAIL_N_BASE, "complexity": FP_FAIL_COMPLEXITY}[kind]
                    ok = v[sel] == (FP_PASS_FILTER if at == 0 else fail)
                elif kind == "cut_front":
                    ok = (front[sel] == want) == (at == 0)
                elif kind == "cut_tail":
                    ok = ((front[sel] + ln[sel]) == want) == (at == 0)
                elif kind == "cut_right":
                    ok = ln[sel] == want
                elif kind == "overlap":
                    if tag == "2":
                        continue
                    hit = (ov["overlapped"][sel] == 1) & (ov["offset"][sel].astype(int) == want)
                    ok = hit == (at == 0)
                elif kind == "polyg":
                    ok = (ln[sel] < want) == (at == 0)
                else:
                    ok = (rec["polyx_len"][sel] > 0) == (at == 0)
                c = out.setdefault(kind, [0, 0, 0, 0])
                c[2 * at] += int(ok.sum())
                c[2 * at + 1] += int(sel.sum())
    return out


# option sets whose threshold reads reach their predicate untouched: the boundary outcomes are asserted on these
THRESHOLD_CHECKS = {
    "filter.unqualified_pct0": ("lowq", "nbase"),
    "filter.unqualified_pct50": ("lowq", "nbase"),
    "filter.unqualified_pct99": ("lowq", "nbase"),
    "filter.avg_qual20": ("avgq",),
    "filter.n_base_limit0": ("nbase",),
    "filter.n_base_limit50": ("nbase",),
    "filter.complexity33": ("complexity",),
    "filter.complexity50": ("complexity",),
    "filter.complexity99": ("complexity",),
    "cut_front_tail.w1_q30": ("cut_front", "cut_tail"),
    "cut_front_tail.w4_q30": ("cut_front", "cut_tail"),
    "cut_front_tail.w33_q1": ("cut_front", "cut_tail"),
    "cut_right.plane4_dp4a.w4_q30": ("cut_right",),
    "cut_right.plane4.w8_q1": ("cut_right",),
    "cut_right.scalar.w9_q30": ("cut_right",),
    "cut_right.scalar.w33_q30": ("cut_right",),
    "polyg.plane.only_min10": ("polyg",),
    "polyg.plane.only_min30": ("polyg",),
    "polyg.plane_off.only_min33": ("polyg",),
    "overlap.threshold": ("overlap",),
}


def threshold_checks(name, S):
    """Predicates whose boundary outcomes are asserted for option set `name` at stride S.  Below a stride of 64 two limits do not fit
    a row: 51 N bases, and a 33-base front window clear of the 33-base tail window."""
    if S < 64 and name in ("filter.n_base_limit50", "cut_front_tail.w33_q1"):
        return ()
    return THRESHOLD_CHECKS.get(name, ())
