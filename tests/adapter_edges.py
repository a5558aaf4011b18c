"""Adapter sequences at every shape the sequence trimmers branch on, and reads planted on both sides of each of their limits (DESIGN §3).

SHAPES holds the adapters: random A/C/G/T at lengths 1-8, 11, 12, 15, 16, 31-33, 63-65, 96, 97, 128, 200 and 255 (the early return
below matchReq, the A-tail starts -2 / -3 / -4 of scan 1, one to eight 32-base plane words, the 64-bit fields of the negative starts
and of the one-gap quick reject up to 64 bases and none from 65 on); homopolymer, period-2 and period-3 adapters; N at the start,
the end and at 31 / 32 / 63 / 64 (the adapter's N plane); a lower-case or IUPAC byte, which takes the byte path.  adapter_cases(paired)
lists named option sets: each shape as adapter_seq_r1 / _r2 ("seq.*") and as a one-entry fasta list ("fasta.*"), fasta lists of
1 / 16 / 17 / 256 / 257 / 512 entries (matchReq 4 / 5 / 6 on both sides of each step) with a repeated entry, a list whose adapters
trim the same read one after another, and reads whose front is moved by trim_front (not a multiple of 32).

case_batch(name, paired, S, seed) plants reads for the adapters of a case (label at = 0 on a limit, at = 1 one past it):
  scan1   the adapter at p = -4 .. -1, 0, 1, 31, 32, 33, rlen - alen, the first tail position and rlen - matchReq - 1 with exactly
          cmplen / 8 mismatches (half of them N), and one more;
  tail    the adapter's first c bases at the read end, c = matchReq + 1 .. min(alen, 32) - 1;
  gap2 / gap3   the adapter with one inserted / one deleted base at the read start, at c == cmax (trim to length 0) with exactly
          c / 8 - 1 mismatches and one more, the mismatches in the first 8k bases for k = 1 .. 8 (gap_below: the gapped adapter
          stops before cmax);
  len     the adapter, then random bases, cut to 0 .. matchReq + 2, 63, 64, 65 and S bases;
  concat  list entries one after another at the read end, in reverse list order (each trims once);
  dimer   pairs whose two reads both start with their adapter.
Pairs hold two unrelated reads (no overlap), so the overlap trimmer leaves them to the sequence trimmers.  boundary_outcomes()
reads the records back and counts, per class, how many reads on each side of the limit came out as that side should."""
import numpy as np

from fastp_b200 import capi

import fp_testlib as T

ACGT = b"ACGT"
LENGTHS = (1, 2, 3, 4, 5, 6, 7, 8, 11, 12, 15, 16, 31, 32, 33, 63, 64, 65, 96, 97, 128, 200, 255)
LIST_SIZES = (1, 16, 17, 256, 257, 512)
KINDS = ("scan1", "tail", "gap2", "gap3", "gap_below", "len", "concat", "dimer", "fill")
K = {k: i for i, k in enumerate(KINDS)}
CHECKED = ("scan1", "tail", "gap2", "gap3")          # classes whose two sides boundary_outcomes() tells apart


def _rand(rng, n):
    return bytes(rng.choice(np.frombuffer(ACGT, np.uint8), n).tobytes()) if n > 0 else b""


def _shapes():
    rng = np.random.default_rng(20261019)
    s = {}
    for L in LENGTHS:
        a = bytearray(_rand(rng, L))
        if L == 64:
            a[63] = ord("G")             # scan 2's field reads read[64] against adapter[63]: a last base other than A tells them apart
        s[f"rand{L}"] = a.decode()
    s["homo16"] = "G" * 16
    s["homo33"] = "C" * 33
    s["per2_64"] = "AC" * 32
    s["per3_33"] = "ACG" * 11
    a = bytearray(_rand(rng, 64)); a[0] = a[63] = ord("N")
    s["n_start_end64"] = a.decode()
    a = bytearray(_rand(rng, 96))
    for i in (31, 32, 63, 64):
        a[i] = ord("N")
    s["n_31_32_63_64_96"] = a.decode()
    a = bytearray(_rand(rng, 33)); a[5] = ord("a")
    s["lower_a33"] = a.decode()
    a = bytearray(_rand(rng, 64)); a[40] = ord("R")
    s["iupac_r64"] = a.decode()
    a = bytearray(_rand(rng, 96)); a[70] = ord("Y")
    s["iupac_y96"] = a.decode()
    return s


SHAPES = _shapes()


def _lists():
    """name -> fasta list.  Entries cycle through the shapes of 6 bases or more (what the reference's fasta loader keeps), the
    second entry repeats the first, and the rest are random adapters of 6-40 bases."""
    rng = np.random.default_rng(7)
    keep = [v for v in SHAPES.values() if len(v) >= 6]
    out = {}
    for n in LIST_SIZES:
        items = []
        for i in range(n):
            if i == 1:
                items.append(items[0])
            elif i < len(keep) and i % 3 == 0:
                items.append(keep[i])
            else:
                items.append(_rand(rng, int(rng.integers(6, 41))).decode())
        out[f"list{n}"] = items
    out["chain5"] = [SHAPES["rand16"], SHAPES["n_start_end64"], SHAPES["rand12"], SHAPES["lower_a33"], SHAPES["rand31"]]
    return out


LISTS = _lists()
FRONTS = {"front5.rand33": (5, "rand33"), "front37.rand64": (37, "rand64"), "front37.rand200": (37, "rand200")}


def adapter_cases(paired):
    """name -> dict(kw=option keywords, plant=[(adapters planted in read 1), (in read 2)], mreq=matchReq of the planted adapters,
    front=trim_front, concat=list planted as concatemers)."""
    cases = {}
    for k, a in SHAPES.items():
        cases[f"seq.{k}"] = dict(kw=dict(adapter_seq_r1=a, adapter_seq_r2=a if paired else None), plant=([a], [a]), mreq=4)
        cases[f"fasta.{k}"] = dict(kw=dict(fasta_adapters=[a]), plant=([a], [a]), mreq=4)
    for k, items in LISTS.items():
        n = len(items)
        mreq = 6 if n > 256 else 5 if n > 16 else 4
        pick = sorted({0, n // 2, n - 1})
        cases[f"fasta.{k}"] = dict(kw=dict(fasta_adapters=items), plant=([items[i] for i in pick], [items[i] for i in pick[::-1]]), mreq=mreq,
                                   concat=[a for a in items[:8] if len(a) <= 40] if k != "chain5" else items)
    for k, (f, shape) in FRONTS.items():
        a = SHAPES[shape]
        cases[k] = dict(kw=dict(adapter_seq_r1=a, adapter_seq_r2=a if paired else None, trim_front1=f, trim_front2=f if paired else 0),
                        plant=([a], [a]), mreq=4, front=f)
    return cases


def case_params(name, paired, lib=None):
    kw = {k: v for k, v in adapter_cases(paired)[name]["kw"].items() if v is not None}
    return capi.default_params(paired, lib=lib or T.oracle(), **kw)


def units_for(name, S):
    """Reads per side: the long lists cost the reference O(list x read length) per read, so they get a few hundred."""
    n = len(adapter_cases(0)[name]["kw"].get("fasta_adapters", ()))
    return 240 if n > 200 else None


# ---------------- planted reads ----------------
def _sub(b, rng, use_n):
    if use_n:
        return ord("N")
    c = ACGT[int(rng.integers(0, 4))]
    while c == b:
        c = ACGT[int(rng.integers(0, 4))]
    return c


def _copy_adapter(a):
    """Adapter bytes as read bases: A/C/G/T/N as they are (N against N is no mismatch), any other byte as a base it differs from."""
    return bytearray(b if b in b"ACGTN" else ord("T") for b in a.encode())


def _mismatch_at(read, a, j, k):
    """read[j] against adapter[k] (bytes compared as the reference compares them)."""
    return read[j] != ord(a[k])


def _scan1_read(a, rlen, p, mm, rng, use_n):
    """Read of rlen bases with adapter a at position p (p < 0: the read starts with a[-p:]) and exactly mm mismatches over the
    compared bases; None if they do not fit."""
    alen = len(a)
    cmplen = min(rlen - p, alen)
    so = max(0, -p)
    read = bytearray(_rand(rng, rlen))
    ad = _copy_adapter(a)
    for k in range(so, cmplen):
        read[p + k] = ad[k]
    cmp = [p + k for k in range(so, cmplen)]
    have = sum(_mismatch_at(read, a, j, j - p) for j in cmp)
    clean = [j for j in cmp if not _mismatch_at(read, a, j, j - p) and a[j - p] != "N"]
    need = mm - have
    if need < 0 or need > len(clean):
        return None
    for i, j in enumerate(rng.choice(clean, need, replace=False) if need else []):
        read[int(j)] = _sub(read[int(j)], rng, use_n and i % 2 == 0)
    return bytes(read)


def _gap_read(a, rlen, scan, c, mm, k8, rng, stop=None):
    """Scan 2 (one base inserted into the read) or scan 3 (one adapter base missing from it): the read starts with the gapped
    adapter, its mismatches against the aligned adapter lie before the gap and in the first max(8 * k8, mm) bases."""
    i = max(2, c // 2 - 3 + k8 % 5)                                     # the gap: far enough from both ends that scan 1 cannot hit
    ad = _copy_adapter(a)
    if scan == 2:
        body = ad[:i] + bytearray(_rand(rng, 1)) + ad[i:]
    else:
        body = ad[:i] + ad[i + 1:]
    if stop is not None:
        body = body[:stop]
    read = bytearray(body[:rlen]) + bytearray(_rand(rng, max(0, rlen - len(body))))
    mm -= sum(b not in "ACGTN" for b in a[:c + (scan == 3)])          # bytes no read base equals are mismatches already
    lim = min(i, max(8 * k8, mm))
    clean = [j for j in range(lim) if a[j] in "ACGT"]
    if mm < 0 or mm > len(clean):
        return None
    for j in (rng.choice(clean, mm, replace=False) if mm else []):
        read[int(j)] = _sub(read[int(j)], rng, False)
    return bytes(read)


class _Side:
    def __init__(self):
        self.rows = []                                 # (seq, kind, at, want)

    def add(self, seq, kind, at, want):
        self.rows.append((bytes(seq), K[kind], at, want))


def _plant_adapter(a, S, mreq, rng, out):
    alen = len(a)
    start = -4 if alen >= 16 else -3 if alen >= 12 else -2 if alen >= 8 else 0
    for rlen in sorted({S, max(1, S - 7)}):
        npos = rlen - mreq
        a0 = min(alen, 32)
        ptail = max(rlen - a0 + 1, 0)
        ps = set(range(start, 0)) | {0, 1, 31, 32, 33, rlen - alen, ptail, rlen - mreq - 1}
        for n, p in enumerate(sorted(x for x in ps if start <= x < npos and x < rlen)):
            cmplen = min(rlen - p, alen)
            if alen < mreq or cmplen <= 0:
                continue
            for at in (0, 1):
                r = _scan1_read(a, rlen, p, cmplen // 8 + at, rng, use_n=n % 2 == 1)
                if r is not None:
                    out.add(r, "scan1", at, 0 if p < 0 else p)
        for c in range(mreq + 1, a0):
            p = rlen - c
            if p < 0 or p >= npos:
                continue
            for at in (0, 1):
                r = _scan1_read(a, rlen, p, c // 8 + at, rng, use_n=False)
                if r is not None:
                    out.add(r, "tail", at, p)
    if alen >= 8:
        for scan in (2, 3):
            for rlen in sorted({S, min(S, alen + (1 if scan == 2 else 0)), min(S, 65)}):
                cmax = min(rlen - 1, alen) if scan == 2 else min(rlen, alen - 1)
                if cmax < 8 or rlen - mreq - (1 if scan == 2 else 0) <= 0:
                    continue
                for k8 in range(1, 9):
                    for at in (0, 1):
                        r = _gap_read(a, rlen, scan, cmax, cmax // 8 - 1 + at, k8, rng)
                        if r is not None:
                            out.add(r, f"gap{scan}", at, 0)
                    stop = cmax - 3 - k8
                    if stop >= 8:
                        r = _gap_read(a, rlen, scan, stop, max(stop // 8 - 1, 0), k8, rng, stop=stop + (1 if scan == 2 else 0))
                        if r is not None:
                            out.add(r, "gap_below", 2, -1)
    tail = _copy_adapter(a) + bytearray(_rand(rng, S))
    for rlen in sorted(set(range(0, mreq + 3)) | {63, 64, 65, S}):
        if rlen <= S:
            out.add(tail[:rlen], "len", 2, -1)


def _plant_concat(items, S, rng, out, n=12):
    body = b"".join(x.encode() for x in reversed(items))
    body = bytes(_copy_adapter(body.decode()))
    for _ in range(n):
        ins = int(rng.integers(0, max(1, S - len(body)) + 1))
        r = (_rand(rng, ins) + body)[:S]
        out.add(r, "concat", 2, -1)


MANY_TRIMS = [bytes(np.random.default_rng(40 + i).choice(np.frombuffer(ACGT, np.uint8), 6)).decode() for i in range(40)]


def many_trims_input(n, lib=None):
    """(params, PE arrays at stride 256): a 40-entry list of 6-mers (matchReq 5) and reads that end in the concatemer of all 40 in
    reverse list order, so most reads are trimmed 30-40 times: up to 82 adapter events per pair."""
    p = capi.default_params(1, lib=lib or T.oracle(), fasta_adapters=MANY_TRIMS)
    import edge_inputs as E
    return p, E.adapter_concatemers(n, 256, MANY_TRIMS, np.random.default_rng(n), 1)


def case_batch(name, paired, S, seed):
    """(arrs, labels, front) at row stride S for case `name`; labels[side] is a structured array (kind, at, want) per unit, want
    being the length the read is trimmed to."""
    case = adapter_cases(paired)[name]
    rng = np.random.default_rng(seed)
    front = case.get("front", 0)
    Se = S - front                                     # the reads' length once trim_front has moved their front
    sides = [_Side(), _Side()] if paired else [_Side()]
    for k, sd in enumerate(sides):
        for a in case["plant"][k]:
            _plant_adapter(a, Se, case["mreq"], rng, sd)
        if case.get("concat"):
            _plant_concat(case["concat"], Se, rng, sd)
    cap = units_for(name, S)
    for sd in sides:
        if cap and len(sd.rows) > cap:
            keep = rng.choice(len(sd.rows), cap, replace=False)
            sd.rows = [sd.rows[i] for i in sorted(keep)]
    if paired:                                         # side 2 shuffled against side 1, then pairs that are both adapter dimers
        a, b = sides
        b.rows = [b.rows[i] for i in rng.permutation(len(b.rows))]
        n = max(len(a.rows), len(b.rows))
        for sd in sides:
            while len(sd.rows) < n:
                rlen = int(rng.integers(0, Se + 1))
                sd.add(_rand(rng, rlen), "fill", 2, -1)
        for _ in range(6):
            for k, sd in enumerate(sides):
                ad = case["plant"][k][0]
                sd.add((bytes(_copy_adapter(ad)) + _rand(rng, Se))[:int(rng.integers(max(1, min(len(ad), Se) // 2), Se + 1))], "dimer", 2, -1)
    n = len(sides[0].rows)
    order = rng.permutation(n)
    _, arrs = capi.host_batch(n, S, 1 if paired else 0)
    lab_dtype = np.dtype([("kind", "i1"), ("at", "i1"), ("want", "<i4")])
    labels = {}
    for k, sd in enumerate(sides):
        tag = str(k + 1)
        lab = np.zeros(n, lab_dtype)
        for r, i in enumerate(order):
            s, kind, at, want = sd.rows[i]
            row = _rand(rng, front) + s
            arrs["seq" + tag][r, :len(row)] = np.frombuffer(row, np.uint8)
            arrs["qual" + tag][r, :len(row)] = rng.integers(33 + 30, 33 + 41, len(row), dtype=np.uint8)
            arrs["len" + tag][r] = len(row)
            lab[r] = (kind, at, want)
        labels[tag] = lab
    return arrs, labels


def boundary_outcomes(labels, res, paired):
    """kind -> [on the limit and trimmed to the planted length, on the limit, one past and not trimmed to it, one past]."""
    out = {}
    for tag in ("1", "2")[: 2 if paired else 1]:
        lab, ln = labels[tag], res["out" + tag]["len"].astype(int)
        for kind in CHECKED:
            for at in (0, 1):
                sel = (lab["kind"] == K[kind]) & (lab["at"] == at)
                if not sel.any():
                    continue
                hit = ln[sel] == lab["want"][sel]
                ok = hit if at == 0 else ~hit
                c = out.setdefault(kind, [0, 0, 0, 0])
                c[2 * at] += int(ok.sum())
                c[2 * at + 1] += int(sel.sum())
    return out


def checked_kinds(name):
    """Classes asserted to land on both sides of their limit in case `name`: those its planted adapters have (scan 1 from matchReq
    bases on, tails from matchReq + 2, scan 2 from 8 and scan 3 from 9), none for homopolymer and periodic adapters (they also match
    themselves shifted, so their reads may trim before the planted position), no tails for lists of hundreds of adapters (some
    entry matches the last 6-7 bases of most random reads)."""
    case = adapter_cases(0)[name]
    alen = min(len(a) for a in case["plant"][0])
    if any(t in name for t in ("homo", "per2", "per3")) or alen < case["mreq"]:
        return ()
    kinds = ["scan1"]
    if min(alen, 32) > case["mreq"] + 1 and not name.startswith(("fasta.list256", "fasta.list257", "fasta.list512")):
        kinds.append("tail")
    if alen >= 8:
        kinds.append("gap2")
    if alen >= 9:
        kinds.append("gap3")
    return tuple(kinds)
