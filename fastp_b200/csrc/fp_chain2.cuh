/*
 * fp_chain2.cuh -- second-generation fused kernel (fp_chain2_kernel).
 *
 * Same tile pipeline as before (TMA bulk loads -> bit planes + validation -> dense column pass), but
 *   * the dense pass gives each thread TWO cycles (half a word column) so only 40 accumulator registers stay
 *     live across the persistent loop, and
 *   * the operator chain runs ONE THREAD PER READ / PAIR on the bit planes: with lo/hi/N/low-quality planes a
 *     150-base read is 5 words, so overlap analysis, adapter scans, the pass/fail filter and base correction are
 *     a few word operations per candidate and a warp handles 32 pairs at once instead of one.  Byte-level work
 *     that is genuinely per base (post-filter statistics of removed / re-added bases) stays warp-cooperative:
 *     lanes flag what they need and the warp walks the flagged lanes.
 * Rows holding bytes outside {A,C,G,T,N} use scalar byte-exact twins of every operator.
 * Reference semantics are cited per operator (file:line under /root/reference/src), as in fp_device.cuh.
 */
#pragma once
#include "fp_device.cuh"

/* unroll factors of the two hottest loops (plane / histogram items, dense column pass) */
#ifndef FP_ITEM_UNROLL
#define FP_ITEM_UNROLL 1
#endif
#ifndef FP_DENSE_UNROLL
#define FP_DENSE_UNROLL 1
#endif
static constexpr int kItemUnroll = FP_ITEM_UNROLL, kDenseUnroll = FP_DENSE_UNROLL;   /* (#pragma unroll does not expand macros) */

/* shared-memory counter += 1 at a 32-bit shared-window address, optionally predicated (no branch, no return value) */
__device__ __forceinline__ void smem_inc(uint32_t addr) { asm volatile("red.shared.add.u32 [%0], 1;" :: "r"(addr) : "memory"); }
/* += 1 iff a > B */
#define smem_inc_gt(addr, a, B) asm volatile("{ .reg .pred p; setp.gt.s32 p, %1, %2; @p red.shared.add.u32 [%0], 1; }" :: "r"(addr), "r"(a), "r"(B) : "memory")

/* thread-level view of one read: its tile row and planes as 32-bit shared-window addresses, the current window.  Addresses rather
   than three generic pointers keep a read at six registers: the PE chain holds two of them across every out-of-line operator. */
struct TRead {
    uint32_t srow;         /* row start in the shared-memory tile; the qualities are c_p.tile * c_p.stride bytes further */
    uint32_t prow;         /* planes of the row: lo = pl, hi = pl+PW, nn = pl+2PW, lq = pl+3PW */
    int front, len;
    bool null, clean;
    __device__ __forceinline__ uint8_t* seq() const { return static_cast<uint8_t*>(__cvta_shared_to_generic(srow)); }
    __device__ __forceinline__ uint8_t* qual() const { return static_cast<uint8_t*>(__cvta_shared_to_generic(srow + (uint32_t)(c_p.tile * c_p.stride))); }
    __device__ __forceinline__ uint32_t* pl() const { return static_cast<uint32_t*>(__cvta_shared_to_generic(prow)); }
};
__device__ __forceinline__ TRead t_read(const uint8_t* seq, const uint32_t* pl, int len, bool clean) {
    TRead r; r.srow = smem_u32(seq); r.prow = smem_u32(pl); r.front = 0; r.len = len; r.null = false; r.clean = clean;
    return r;
}

__device__ __forceinline__ uint32_t tp_bits(const uint32_t* P, int bit) {      /* 32 bits of a plane starting at `bit` */
    const int w = bit >> 5;
    return __funnelshift_r(P[w], P[w + 1], bit & 31);
}

__device__ __forceinline__ uint32_t tp_bits_z(const uint32_t* P, int s0) {   /* tp_bits with zeros below bit 0 */
    if (s0 >= 0) return tp_bits(P, s0);
    if (s0 > -32) return P[0] << (-s0);
    return 0u;
}

/* A read / pair is served by a GROUP of g adjacent lanes (g = 4 for PE, 2 for SE): all lanes run the scalar operators
 * redundantly (same shared-memory addresses -> broadcasts), the long candidate scans (overlap offsets, adapter
 * positions) are split round-robin over the g lanes and combined with group_min, and every side effect (atomics,
 * stores) is done by the group's lane 0 only. */
__device__ __forceinline__ unsigned group_mask(int g) { return (g >= 32 ? 0xffffffffu : ((1u << g) - 1u)) << (lane_id() & ~(g - 1)); }
__device__ __forceinline__ int group_min(int v, int g) {
    const unsigned gm = group_mask(g);          /* only the group's lanes take part: groups of one warp may diverge */
    for (int o = g >> 1; o > 0; o >>= 1) v = min(v, __shfl_xor_sync(gm, v, o));
    return v;
}
/* value of `v` held by the lane of my group for which `mine` is true (exactly one lane, or none -> returns own v) */
__device__ __forceinline__ int group_pick(int v, bool mine, int g) {
    const unsigned gm = group_mask(g);
    const unsigned b = __ballot_sync(gm, mine);
    const int src = b ? __ffs(b) - 1 : lane_id();
    return __shfl_sync(gm, v, src);
}

/* ------------------------------------------------------------------------------------------------
 * Filter::trimAndCut  (filter.cpp:68-207), scalar per thread.  Returns the new window as front | len << 16, or -1 for NULL
 * (a packed value rather than reference outputs: the caller's read state stays in registers across the call).
 * ------------------------------------------------------------------------------------------------ */
__device__ __forceinline__ int tc_pack(int front, int len) { return front | (len << 16); }
__device__ __forceinline__ void tc_apply(TRead& r, int tc) { r.null = tc < 0; if (tc >= 0) { r.front = tc & 0xFFFF; r.len = tc >> 16; } }
__device__ __noinline__ int t_trim_and_cut(const uint8_t* seq, const uint8_t* qualu, int l0, int front, int tail, int sub, int g, const uint32_t* cqp) {
    FP_SMEM(seq);    FP_SMEM(qualu);    FP_SMEM(cqp);
    const bool anycut = c_p.cut_front || c_p.cut_tail || c_p.cut_right;
    if (front == 0 && tail == 0 && !anycut) return tc_pack(0, l0);        /* :71-72 */
    int rlen = l0 - front - tail;                                         /* :75 */
    if (rlen < 0) return -1;
    if (!anycut) return tc_pack(front, rlen);                             /* :79-89 (front==0: resize only) */
    const int l = l0;
    const signed char* q = reinterpret_cast<const signed char*>(qualu);
    if (c_p.cut_front) {                                                  /* :97-127 */
        const int w = c_p.cf_w;
        int s = front;
        if (l - front - tail - w <= 0) return -1;
        int total = 0;
        for (int i = 0; i < w - 1; i++) total += q[s + i];
        for (s = front; s + w < l - tail; s++) {
            total += q[s + w - 1];
            if (s > front) total -= q[s - 1];
            if (total >= c_p.cf_thr) break;
        }
        if (s > 0) s = s + w - 1;
        while (s < l && seq[s] == 'N') s++;
        front = s;
        rlen = l - front - tail;
    }
    if (c_p.cut_right) {                                                  /* :130-163 */
        const int w = c_p.cr_w;
        int s = front;
        if (l - front - tail - w <= 0) return -1;
        bool found = false;
        if (cqp && w <= 8 && c_p.cr_q >= 0 && c_p.cr_q <= 127) {
            /* plane 4 marks the bases below the per-base threshold 33+Q; a window without one sums to at least w*(33+Q).  So only windows
               holding a marked base are summed -- none at all for most reads.  Every lane of the group walks the plane words in the
               reference's order and takes the candidate starts congruent to its own index (a low-quality stretch is shared evenly);
               one vote per word. */
            const int smax = l - tail - w;                                /* window starts s in [front, smax) */
            const int thr = c_p.cr_thr;
            const unsigned gm = group_mask(g);
            const uint32_t share = (g == 4 ? 0x11111111u : g == 2 ? 0x55555555u : 0xFFFFFFFFu) << (g <= 4 ? sub : 0);
            int best = 1 << 20;
            for (int wb = front >> 5; 32 * wb < smax; wb++) {
                int mine = 1 << 20;
                const uint32_t c0 = cqp[wb], c1 = cqp[wb + 1];
                uint32_t cand = c0;
                for (int k = 1; k < w; k++) cand |= __funnelshift_r(c0, c1, k);
                cand &= low_mask(smax - 32 * wb) & ~low_mask(front - 32 * wb);
                if (g > 4) { if (sub) cand = 0; } else cand &= share;
                while (cand) {
                    const int sk = 32 * wb + __ffs(cand) - 1;
                    cand &= cand - 1;
                    int tot = 0;
                    if (w == 4) tot = __dp4a((int)ld_u32_unaligned(qualu + sk), 0x01010101, 0);     /* qualities < 128 on clean rows */
                    else for (int k = 0; k < w; k++) tot += q[sk + k];
                    if (tot < thr) { mine = sk; break; }
                }
                if (__any_sync(gm, mine != (1 << 20))) { best = group_min(mine, g); break; }
            }
            if (best < (1 << 20)) { found = true; s = best; }
        } else if (w == 4) {
            /* window of 4 = one 32-bit field: the group's lanes take consecutive aligned words (4 window starts each), the window sum is
               one dp4a; rounds advance together so the group-min picks the first start in the reference's order */
            const int smax = l - tail - w;                                /* window starts s in [front, smax) */
            const int thr = c_p.cr_thr;
            const unsigned gm = group_mask(g);
            int best = 1 << 20;
            for (int wb = (front >> 2) + sub; (wb - sub) * 4 < smax; wb += g) {
                const int b0 = wb * 4;
                int mine = 1 << 20;
                if (b0 < smax) {
                    const uint32_t W0 = *reinterpret_cast<const uint32_t*>(qualu + b0), W1 = *reinterpret_cast<const uint32_t*>(qualu + b0 + 4);
                    #pragma unroll
                    for (int k = 3; k >= 0; k--) {
                        const int sk = b0 + k;
                        const int tot = __dp4a((int)__funnelshift_r(W0, W1, 8 * k), 0x01010101, 0);       /* signed chars, like the reference's char sum */
                        if (sk >= front && sk < smax && tot < thr) mine = sk;
                    }
                }
                if (__any_sync(gm, mine != (1 << 20))) { best = group_min(mine, g); break; }   /* one vote per round; the min only when someone hit */
            }
            if (best < (1 << 20)) { found = true; s = best; }
        } else {
            int total = 0;
            for (int i = 0; i < w - 1; i++) total += q[s + i];
            for (s = front; s + w < l - tail; s++) {
                total += q[s + w - 1];
                if (s > front) total -= q[s - 1];
                if (total < c_p.cr_thr) { found = true; break; }
            }
        }
        if (found) {
            while (s < l - 1 && q[s] >= c_p.cr_q) s++;
            rlen = s - front;
        }
    }
    if (!c_p.cut_right && c_p.cut_tail) {                                 /* :166-194 */
        const int w = c_p.ct_w;
        if (l - front - tail - w <= 0) return -1;
        int total = 0;
        int t = l - tail - 1;
        for (int i = 0; i < w - 1; i++) total += q[t - i];
        for (t = l - tail - 1; t - w >= front; t--) {
            total += q[t - w + 1];
            if (t < l - tail - 1) total -= q[t + 1];
            if (total >= c_p.ct_thr) break;
        }
        if (t < l - 1) t = t - w + 1;
        while (t >= 0 && seq[t] == 'N') t--;
        rlen = t - front + 1;
    }
    if (rlen <= 0 || front >= l - 1) return -1;                        /* :196-197 */
    return tc_pack(front, rlen);
}

/* Plane tests that settle the usual case of the two poly-tail trimmers without walking the tail (clean rows only).
 * trimPolyG (polyx.cpp:16-42) trims only if its scan gets past index minLen-1; more than five non-G among the last minLen bases
 * stop it before that (`mismatch > 5`), and so does a read shorter than minLen.
 * trimPolyX (:49-116) with minLen >= 10 cannot stop before pos 8 and trims only if it stops at pos+1 >= minLen: if no base (N counts
 * for every base) fills 8 of the last 9 positions, `needToBreak` holds at pos 8 and the scan ends there without trimming. */
__device__ __forceinline__ bool t_polyg_cannot_trim(const TRead& r, int PW, int minLen) {
    if (r.len < minLen) return true;
    if (!r.clean || minLen > 32 || minLen < 1) return false;
    const int bit = r.front + r.len - minLen;
    const uint32_t g = tp_bits(r.pl(), bit) & tp_bits(r.pl() + PW, bit);           /* G: code 3 (lo = hi = 1; both 0 under N) */
    return __popc(~g & low_mask(minLen)) > 5;
}
__device__ __forceinline__ bool t_polyx_cannot_trim(const TRead& r, int PW, int minLen) {
    if (minLen < 10) return false;
    if (r.len < 9) return true;
    if (!r.clean) return false;
    const int bit = r.front + r.len - 9;
    const uint32_t lo = tp_bits(r.pl(), bit), hi = tp_bits(r.pl() + PW, bit), nn = tp_bits(r.pl() + 2 * PW, bit), m = 0x1FFu;
    const int cA = __popc((~lo & ~hi) & m), cC = __popc((lo & ~hi | nn) & m), cT = __popc((~lo & hi | nn) & m), cG = __popc((lo & hi | nn) & m);
    /* ~lo & ~hi is A or N (both planes are 0 under N): already counts N for A */
    return max(max(cA, cC), max(cT, cG)) <= 7;
}

/* PolyX::trimPolyG  (polyx.cpp:16-42): returns the new length */
__device__ __noinline__ int t_trim_polyg(const uint8_t* data, int rlen, int minLen) {
    FP_SMEM(data);
    int mismatch = 0, i = 0, firstGPos = rlen - 1;
    for (i = 0; i < rlen; i++) {
        if (data[rlen - i - 1] != 'G') mismatch++; else firstGPos = rlen - i - 1;
        const int allowed = (i + 1) / 8;
        if (mismatch > 5 || (mismatch > allowed && i >= minLen - 1)) break;
    }
    if (i >= minLen && firstGPos >= 0 && firstGPos <= rlen) return firstGPos;
    return rlen;
}

/* trimPolyG on the planes (clean rows): the scan's state only changes at non-G bases, so hop from one to the next (at most six before
 * `mismatch > 5` ends it) instead of walking every base.  i counts from the tail (base rlen-1-i); on a run of G's with m mismatches behind it
 * the stop condition `m > (i+1)/8 && i >= minLen-1` holds exactly for max(run start, minLen-1) <= i <= 8m-2. */
__device__ __noinline__ int t_trim_polyg_planes(const uint32_t* pl, int PW, int front, int rlen, int minLen) {
    FP_SMEM(pl);
    auto ng_word = [&](int w) -> uint32_t {                                 /* bit t: base i = 32w + t is not G (valid i only) */
        const int bit = front + rlen - 32 * (w + 1);
        const uint32_t g = __brev(tp_bits_z(pl, bit) & tp_bits_z(pl + PW, bit));
        return ~g & low_mask(rlen - 32 * w);
    };
    int i = 0, m = 0, lastG = -1, brk = -1;
    #pragma unroll 1
    while (i < rlen) {
        int w = i >> 5;
        uint32_t x = ng_word(w) & ~low_mask(i & 31);
        while (!x && 32 * (w + 1) < rlen) { w++; x = ng_word(w); }
        const int nxt = x ? 32 * w + __ffs(x) - 1 : rlen;                  /* next non-G at or after i */
        if (nxt > i) {                                                     /* G's on [i, nxt-1] */
            const int ib = max(i, minLen - 1);
            if (m > 0 && ib <= min(nxt - 1, 8 * m - 2)) { brk = ib; lastG = ib; break; }
            lastG = nxt - 1;
        }
        if (nxt >= rlen) break;
        m++;
        if (m > 5 || (m > (nxt + 1) / 8 && nxt >= minLen - 1)) { brk = nxt; break; }
        i = nxt + 1;
    }
    const int iend = brk >= 0 ? brk : rlen;
    const int firstGPos = lastG >= 0 ? rlen - 1 - lastG : rlen - 1;
    if (iend >= minLen && firstGPos >= 0 && firstGPos <= rlen) return firstGPos;
    return rlen;
}

/* PolyX::trimPolyX  (polyx.cpp:49-116): 0 if addPolyXTrimmed is not called, else px_pack(new length, polyX base, trimmed count) */
__device__ __forceinline__ uint32_t px_pack(int newLen, int poly, int n) { return 0x80000000u | (uint32_t)newLen | ((uint32_t)poly << 12) | ((uint32_t)n << 16); }
__device__ __forceinline__ int px_len(uint32_t t) { return (int)(t & 0xFFFu); }
__device__ __forceinline__ int px_base(uint32_t t) { return (int)((t >> 12) & 3u); }
__device__ __forceinline__ int px_n(uint32_t t) { return (int)((t >> 16) & 0x7FFFu); }
__device__ __noinline__ uint32_t t_trim_polyx(const uint8_t* data, int rlen, int minLen) {
    FP_SMEM(data);
    int a = 0, t = 0, c = 0, g = 0, pos = 0;
    for (pos = 0; pos < rlen; pos++) {
        const uint8_t ch = data[rlen - pos - 1];
        const int n = (ch == 'N');
        a += (ch == 'A') | n; t += (ch == 'T') | n; c += (ch == 'C') | n; g += (ch == 'G') | n;
        const int cmp = pos + 1;
        const int allowed = min(5, cmp / 8);
        const bool need = (cmp - a > allowed) && (cmp - t > allowed) && (cmp - c > allowed) && (cmp - g > allowed);
        if (need && (pos >= 8 || pos + 1 >= minLen - 1)) break;
    }
    if (pos + 1 >= minLen) {
        int poly = 0, mx = a;
        if (t > mx) { mx = t; poly = 1; }
        if (c > mx) { mx = c; poly = 2; }
        if (g > mx) { mx = g; poly = 3; }
        const uint8_t pb = poly == 0 ? 'A' : poly == 1 ? 'T' : poly == 2 ? 'C' : 'G';
        for (;;) {                                                        /* :107-108; data[-1] / data[rlen] never match */
            const int idx = rlen - pos - 1;
            const uint8_t ch = (idx < 0 || idx >= rlen) ? 0 : data[idx];
            if (ch != pb && pos >= 0) pos--; else break;
        }
        const int nl = rlen - pos - 1;
        return px_pack(nl >= 0 && nl <= rlen ? nl : rlen, poly, pos + 1);
    }
    return 0u;
}

/* ------------------------------------------------------------------------------------------------
 * OverlapAnalysis::analyze  (overlapanalysis.cpp:17-146) on bit planes, one thread per pair, no scratch.
 * rc(r2)[k] = complement(row2[e-k]), e = front2+len2-1:  a 32-bit field of rc(r2) is the bit-reversal of a field
 * of row2's planes (complement flips code bit 1, N stays N).
 *   forward  offset o: r1[o+k] vs rc(r2)[k], k < pp  -> r1 field at a moving position vs two constant rc words
 *   backward offset o: r1[k] vs rc(r2)[o+k]          -> equivalently comp(r1[pp-1-t]) vs row2[s+t], s = e-o-pp+1:
 *                      the reversed-complemented r1 prefix Y is constant, row2's field moves (never negative).
 * ------------------------------------------------------------------------------------------------ */
__device__ __forceinline__ unsigned long long tp_bits64(const uint32_t* P, int bit) {
    const int w = bit >> 5, sh = bit & 31;
    const uint32_t lo = __funnelshift_r(P[w], P[w + 1], sh), hi = __funnelshift_r(P[w + 1], P[w + 2], sh);
    return ((unsigned long long)hi << 32) | lo;
}
__device__ __forceinline__ unsigned long long mask64(int n) { return n >= 64 ? ~0ull : (n <= 0 ? 0ull : ((1ull << n) - 1ull)); }

/* Exact no-gap acceptance test of ONE candidate (overlapanalysis.cpp:34-44): mismatches over the protected prefix
 * pp = min(ol, 50) on the three planes; returns the count if it is within lut[ol], else -1.  The 64-base constant side of the
 * comparison (K*) is prepared once per pair and direction by every lane together (OvConst); only the few survivors of the
 * one-plane filter below (and candidates of pairs too short for it) get here, so the divergent part is three plane fields. */
struct OvPlanes { const uint32_t *alo, *ahi, *ann, *plo, *phi, *pnn; int f1, len1, e, len2; };
struct OvConst { unsigned long long klo, khi, knn; };

__device__ __forceinline__ OvConst t_ov_const(const OvPlanes& P, int dir) {
    OvConst K;
    if (dir == 0) {                                                        /* rc(r2)[0..64): reversed tail of r2, hi complemented */
        K.knn = ((unsigned long long)__brev(tp_bits_z(P.pnn, P.e - 63)) << 32) | __brev(tp_bits_z(P.pnn, P.e - 31));
        K.klo = ((unsigned long long)__brev(tp_bits_z(P.plo, P.e - 63)) << 32) | __brev(tp_bits_z(P.plo, P.e - 31));
        K.khi = ~(((unsigned long long)__brev(tp_bits_z(P.phi, P.e - 63)) << 32) | __brev(tp_bits_z(P.phi, P.e - 31))) & ~K.knn;
    } else {                                                               /* Y50[t] = comp(r1[49-t]) */
        const unsigned long long a_nn = tp_bits64(P.ann, P.f1), a_lo = tp_bits64(P.alo, P.f1), a_hi = tp_bits64(P.ahi, P.f1);
        K.knn = __brevll(a_nn) >> 14; K.klo = __brevll(a_lo) >> 14; K.khi = ~(__brevll(a_hi) >> 14) & ~K.knn;
    }
    return K;
}

__device__ __forceinline__ int t_ov_exact(const OvPlanes& P, const OvConst& K, int dir, int o, const int16_t* lut, int& olOut) {
    int ol, bit, sh;
    if (dir == 0) { ol = min(P.len1 - o, P.len2); bit = P.f1 + o; sh = 0; }                       /* r1[o+k] vs rc(r2)[k] */
    else { ol = min(P.len1, P.len2 - o); const int pp = min(ol, 50); bit = P.e - o - pp + 1; sh = 50 - pp; }   /* comp(r1[pp-1-t]) vs row2[bit+t] */
    const uint32_t *Mlo = dir == 0 ? P.alo : P.plo, *Mhi = dir == 0 ? P.ahi : P.phi, *Mnn = dir == 0 ? P.ann : P.pnn;
    const unsigned long long x = (tp_bits64(Mlo, bit) ^ (K.klo >> sh)) | (tp_bits64(Mhi, bit) ^ (K.khi >> sh)) | (tp_bits64(Mnn, bit) ^ (K.knn >> sh));
    const int mm = __popcll(x & mask64(min(ol, 50)));
    olOut = ol;
    return mm <= (int)lut[ol] ? mm : -1;
}

/* One 32-candidate word of the one-plane filter: bit sh of the result is set iff the field at bit offset sh of the word pair
 * (W0, W1) differs from C in at most thr-1 of the positions M keeps.  The plane is X = lo ^ hi (A,G -> 0; C,T -> 1; N -> 0): two
 * bases whose X bits differ are different bases, so this count never exceeds the true mismatch count of the candidate's first
 * F compared bases; every acceptance limit is <= diffLimit, hence a candidate whose count exceeds diffLimit cannot be accepted.
 * X (not lo or hi alone) because a base and its complement always differ in X: reads that end in the same homopolymer or
 * adapter run -- the common non-random case -- do not flood the filter.  Fully unrolled, five instructions per candidate
 * (shift, xor-and, popc, subtract, shift-in of the sign bit), no branches, so the 32 lanes stay together. */
__device__ __forceinline__ uint32_t t_ov_word_hits(uint32_t W0, uint32_t W1, uint32_t C, uint32_t M, int thr) {
    uint32_t hits = 0;
    #pragma unroll
    for (int sh = 31; sh >= 0; sh--) {
        const int t = __popc((__funnelshift_r(W0, W1, sh) ^ C) & M) - thr;      /* negative iff the candidate survives */
        hits = __funnelshift_l((uint32_t)t, hits, 1);                           /* hits = hits << 1 | sign(t) */
    }
    return hits;
}

__device__ __noinline__ fp_ov_result t_analyze_planes(const TRead r1, const TRead r2, int PW, const int16_t* lut, int sub, int g) {
    FP_SMEM(r1.pl());    FP_SMEM(r2.pl());    FP_SMEM(lut);
    OvPlanes P;
    P.alo = r1.pl(); P.ahi = r1.pl() + PW; P.ann = r1.pl() + 2 * PW;
    P.plo = r2.pl(); P.phi = r2.pl() + PW; P.pnn = r2.pl() + 2 * PW;
    P.f1 = r1.front; P.len1 = r1.len; P.len2 = r2.len; P.e = r2.front + r2.len - 1;
    const int len1 = r1.len, len2 = r2.len, f1 = r1.front, e = P.e;
    const int req = c_p.ov_require;
    const int Fmax = min(32, max(req, 1));       /* bases the filter looks at: every candidate's overlap is longer than req ... */
    fp_ov_result ov; ov.overlapped = 0; ov.has_gap = 0; ov.offset = 0; ov.overlap_len = 0; ov.diff = 0;
    int found_dir = -1, found_o = 0, found_mm = 0, found_ol = 0;
    #pragma unroll 1
    for (int dir = 0; dir < 2 && found_dir < 0; dir++) {
        /* candidates o = 0 .. ncand-1 in the reference's order (:48-65 forward, :73-89 backward).  When the fixed read has at least F
           bases, the first F compared bases of candidate o are an F-bit field of the MOVING read's X plane against a constant:
             forward   r1 field at bit f1+o          vs  C = rc(r2)[0..F)  = reversed last F bases of r2 (complement flips X, so ~)
             backward  r2 field at bit e-(F-1)-o     vs  C = reversed complemented r1[0..F)   (bit t of the field is rc(r2)[o+F-1-t])
           The group's lanes take whole plane words (32 consecutive candidates each) in the order of increasing o. */
        const int ncand = dir == 0 ? len1 - req : len2 - req;
        const int lfix = dir == 0 ? len2 : len1, lmov = dir == 0 ? len1 : len2;
        /* ... unless the fixed read itself is shorter (quality trimming): then every candidate overlaps all of it.  The acceptance limit
           grows with the overlap length, so the largest overlap of this direction bounds them all. */
        const int F = min(Fmax, lfix);
        const uint32_t FM = low_mask(F);
        const int thr = (int)lut[min(lmov, lfix)] + 1;
        const int nscan = F >= 1 ? max(ncand, 0) : 0;
        int my_o = 1 << 20, my_mm = 0, my_ol = 0;
        const OvConst K = t_ov_const(P, dir);
        if (nscan > 0) {
            const uint32_t *Mlo = dir == 0 ? P.alo : P.plo, *Mhi = dir == 0 ? P.ahi : P.phi;
            /* X of the complement is ~X, except under N (0 either way; lo = hi = 0 under N in the planes) */
            uint32_t C;
            if (dir == 0) { const int s0 = e - 31; C = __brev(~(tp_bits_z(P.plo, s0) ^ tp_bits_z(P.phi, s0)) & ~tp_bits_z(P.pnn, s0)); }
            else C = __brev(~(tp_bits(P.alo, f1) ^ tp_bits(P.ahi, f1)) & ~tp_bits(P.ann, f1)) >> (32 - F);
            const int blo = dir == 0 ? f1 : e - (F - 1) - (nscan - 1), bhi = dir == 0 ? f1 + nscan - 1 : e - (F - 1);   /* field starts */
            const int wlo = blo >> 5, whi = bhi >> 5;
            #pragma unroll 1
            for (int wi = sub; wi <= whi - wlo && my_o == (1 << 20); wi += g) {
                const int w = dir == 0 ? wlo + wi : whi - wi;
                const uint32_t W0 = Mlo[w] ^ Mhi[w], W1 = Mlo[w + 1] ^ Mhi[w + 1];
                uint32_t hits = t_ov_word_hits(W0, W1, C, FM, thr);
                hits &= low_mask(bhi - 32 * w + 1) & ~low_mask(blo - 32 * w);
                /* survivors (the true overlap, rarely anything else): exact test in the reference's order.  Lanes with survivors reach
                   this loop together, so the warp pays the test once per round, not once per survivor. */
                while (hits) {
                    const int sh = dir == 0 ? __ffs(hits) - 1 : 31 - __clz(hits);
                    hits &= ~(1u << sh);
                    const int bit = 32 * w + sh;
                    const int o = dir == 0 ? bit - f1 : e - (F - 1) - bit;
                    int ol;
                    const int mm = t_ov_exact(P, K, dir, o, lut, ol);
                    if (mm >= 0) { my_o = o; my_mm = mm; my_ol = ol; break; }
                }
            }
        } else {
            #pragma unroll 1
            for (int o = sub; o < ncand; o += g) {           /* fixed read shorter than the filter: exact test of every candidate */
                int ol;
                const int mm = t_ov_exact(P, K, dir, o, lut, ol);
                if (mm >= 0) { my_o = o; my_mm = mm; my_ol = ol; break; }
            }
        }
        const int best = group_min(my_o, g);
        if (best < (1 << 20)) {
            found_dir = dir; found_o = best;
            found_mm = group_pick(my_mm, my_o == best, g); found_ol = group_pick(my_ol, my_o == best, g);
        }
    }
    if (found_dir >= 0) {
        int diff = found_mm;
        if (found_ol > 50) {                                               /* :41-43 full recount over the whole overlap */
            diff = 0;
            const int abit = f1 + (found_dir == 0 ? found_o : 0), bbit = found_dir == 0 ? 0 : found_o;
            for (int k = 0; k * 32 < found_ol; k++) {
                const int s0 = e - (bbit + 32 * k) - 31;
                const uint32_t rn = __brev(tp_bits_z(P.pnn, s0));
                const uint32_t rl_ = __brev(tp_bits_z(P.plo, s0)), rh = ~__brev(tp_bits_z(P.phi, s0)) & ~rn;
                const uint32_t x = (tp_bits(P.alo, abit + 32 * k) ^ rl_) | (tp_bits(P.ahi, abit + 32 * k) ^ rh) | (tp_bits(P.ann, abit + 32 * k) ^ rn);
                diff += __popc(x & low_mask(found_ol - 32 * k));
            }
        }
        ov.overlapped = 1; ov.offset = (int16_t)(found_dir == 0 ? found_o : -found_o); ov.overlap_len = (int16_t)found_ol; ov.diff = (int16_t)diff;
    }
    return ov;
}

/* byte-exact twin for rows with bytes outside {A,C,G,T,N} */
__device__ __noinline__ fp_ov_result t_analyze_bytes(const TRead r1, const TRead r2, const int16_t* lut) {
    FP_SMEM(r1.seq());    FP_SMEM(r2.seq());    FP_SMEM(lut);
    const uint8_t* s1 = r1.seq() + r1.front; const uint8_t* s2 = r2.seq() + r2.front;
    const int len1 = r1.len, len2 = r2.len, req = c_p.ov_require;
    fp_ov_result ov; ov.overlapped = 0; ov.has_gap = 0; ov.offset = 0; ov.overlap_len = 0; ov.diff = 0;
    for (int dir = 0; dir < 2; dir++) {
        const int ncand = dir == 0 ? len1 - req : len2 - req;
        for (int o = 0; o < ncand; o++) {
            const int ol = dir == 0 ? min(len1 - o, len2) : min(len1, len2 - o);
            const int limit = lut[ol], pp = min(ol, 50);
            int mm = 0;
            for (int k = 0; k < pp; k++) {
                const uint8_t a = dir == 0 ? s1[o + k] : s1[k];
                const uint8_t b = dev_complement(dir == 0 ? s2[len2 - 1 - k] : s2[len2 - 1 - o - k]);
                mm += (a != b);
            }
            if (mm <= limit) {
                int diff = mm;
                if (ol > 50) {
                    diff = 0;
                    for (int k = 0; k < ol; k++) {
                        const uint8_t a = dir == 0 ? s1[o + k] : s1[k];
                        const uint8_t b = dev_complement(dir == 0 ? s2[len2 - 1 - k] : s2[len2 - 1 - o - k]);
                        diff += (a != b);
                    }
                }
                ov.overlapped = 1; ov.offset = (int16_t)(dir == 0 ? o : -o); ov.overlap_len = (int16_t)ol; ov.diff = (int16_t)diff;
                return ov;
            }
        }
    }
    return ov;
}

/* ------------------------------------------------------------------------------------------------
 * The one-gap passes of OverlapAnalysis::analyze (overlapanalysis.cpp:91-139, --allow_gap_overlap_trimming) with
 * Matcher::diffWithOneInsertion (matcher.cpp:56-100) in closed form: with D1[j] = ins[j]!=norm[j], D2[j] = ins[j+1]!=norm[j]
 * and prefix sums P1/P2 it returns -1 when P1[c-1] + D2[c-1] > limit, else min_{1<=i<=c-1}(P1[i]-P2[i]) + P2[c]
 * (the early breaks / sentinel never change an accepted value, cf. tests/test_closed_forms.py).  Byte-level, one
 * sequential scan per (offset, orientation) with an early reject on the lower bound sum(D1 & D2); rare option, kept simple.
 * ------------------------------------------------------------------------------------------------ */
template <class FI, class FN>
__device__ __forceinline__ int t_diff_one_insertion(FI ins, FN norm, int c, int limit) {
    int p1 = 0, p2 = 0, runmin = 1 << 20, lb = 0, p1cm1 = 0, d2last = 0;
    for (int j = 0; j < c; j++) {
        const uint8_t nj = norm(j);
        const int d1 = ins(j) != nj, d2 = ins(j + 1) != nj;
        lb += d1 & d2;
        if (lb > limit) return 1 << 20;                                   /* every split costs at least lb */
        p1 += d1; p2 += d2;
        if (j + 1 <= c - 1) runmin = min(runmin, p1 - p2);
        if (j == c - 2) p1cm1 = p1;
        if (j == c - 1) d2last = d2;
    }
    if (c >= 2 && p1cm1 + d2last > limit) return -1;
    return runmin + p2;
}

__device__ __noinline__ fp_ov_result t_analyze_gap(const TRead r1, const TRead r2, const int16_t* lut, int sub, int g) {
    FP_SMEM(r1.seq());    FP_SMEM(r2.seq());    FP_SMEM(lut);
    const uint8_t* s1 = r1.seq() + r1.front; const uint8_t* s2 = r2.seq() + r2.front;
    const int len1 = r1.len, len2 = r2.len, req = c_p.ov_require;
    fp_ov_result ov; ov.overlapped = 0; ov.has_gap = 0; ov.offset = 0; ov.overlap_len = 0; ov.diff = 0;
    for (int dir = 0; dir < 2; dir++) {
        const int ncand = dir == 0 ? len1 - req : len2 - req;
        int my_o = 1 << 20, my_d = 0, my_ol = 0;
        for (int o = sub; o < ncand; o += g) {
            const int ol = dir == 0 ? min(len1 - o, len2) : min(len1, len2 - o);
            const int limit = lut[ol], c = ol - 1;
            const int ao = dir == 0 ? o : 0, bo = dir == 0 ? 0 : o;       /* str1 + ao  vs  rc(r2) + bo */
            auto A = [&](int j) -> uint8_t { return s1[ao + j]; };
            auto B = [&](int j) -> uint8_t { return dev_complement(s2[len2 - 1 - bo - j]); };
            int d = t_diff_one_insertion(A, B, c, limit);
            if (d < 0 || d > limit) d = t_diff_one_insertion(B, A, c, limit);
            if (d <= limit && d >= 0) { my_o = o; my_d = d; my_ol = ol; break; }
        }
        const int best = group_min(my_o, g);
        if (best < (1 << 20)) {
            ov.overlapped = 1; ov.has_gap = 1; ov.offset = (int16_t)(dir == 0 ? best : -best);
            ov.diff = (int16_t)group_pick(my_d, my_o == best, g); ov.overlap_len = (int16_t)group_pick(my_ol, my_o == best, g);
            return ov;
        }
    }
    return ov;
}

/* Effect of ONE corrected base on the post-filter statistics, in full-read context (cycle = row position P, 5-mers of
 * the whole original row): -(old base, old quality) +(new base, new quality).  The dense pass credited the ORIGINAL row to
 * pre and post; with this delta the block-private (or, for unclean rows, global) post accumulators describe the CURRENT row,
 * so the end-of-chain tail/whole-read removal can use the current bytes for corrected and uncorrected reads alike.
 * Called by one thread while seq[P] still holds the old base. */
__device__ __noinline__ void t_patch_delta(const DeltaAcc D, unsigned long long* G, bool clean, int side, const uint8_t* seq, int l0, int P,
                                           uint8_t ob, uint8_t oq, uint8_t nb, uint8_t nq) {
    FP_SMEM(D.cyc);    FP_SMEM(D.kmer);    FP_SMEM(D.qh);    FP_SMEM(seq);
    const fp_counter_layout& L = c_p.L;
    #pragma unroll 1
    for (int pass = 0; pass < 2; pass++) {
        const uint8_t b = pass ? nb : ob, q = pass ? nq : oq;
        const int sg = pass ? +1 : -1;
        if (clean) {
            if (q < FP_QUAL_BINS) atomicAdd(&D.qh[side * FP_QUAL_BINS + q], sg);
            if (P < D.cycles) {
                int* c4 = D.cyc + side * D.cycles * 20 + (P * 5 + ((0x43F21F0Fu >> (4 * (b & 7))) & 0xF)) * 4;
                atomicAdd(&c4[0], sg);
                if (q >= '5') atomicAdd(&c4[1], sg);
                if (q >= '?') atomicAdd(&c4[2], sg);
                atomicAdd(&c4[3], sg * ((int)q - 33));
            }
        } else {
            const unsigned long long one = (unsigned long long)(long long)sg;
            const int st = side * 2 + 1, bb = b & 7;
            if (q < FP_QUAL_BINS) red_add64(&G[fp_off_qualhist(&L, st, q)], one);
            if (P < L.cycles) {
                if (q >= '?') { red_add64(&G[fp_off_cycle(&L, st, 0 * 8 + bb, P)], one); red_add64(&G[fp_off_cycle(&L, st, 1 * 8 + bb, P)], one); }
                else if (q >= '5') red_add64(&G[fp_off_cycle(&L, st, 1 * 8 + bb, P)], one);
                red_add64(&G[fp_off_cycle(&L, st, 2 * 8 + bb, P)], one);
                red_add64(&G[fp_off_cycle(&L, st, 3 * 8 + bb, P)], (unsigned long long)((long long)sg * ((int)q - 33)));
            }
        }
        /* 5-mers ending at i = P .. P+4 (stats.cpp:228-266) with the base at P set to b.  The block-private table is indexed like the
           pre-filter one (oldest base in the low digit, codes A0 C1 T2 G3; mapped to the reference's index at the flush). */
        #pragma unroll 1
        for (int i = max(P, 4); i <= min(P + 4, l0 - 1); i++) {
            int code = 0, field = 0; bool ok = true;
            #pragma unroll
            for (int k = 0; k < 5; k++) {
                const int pos = i - 4 + k;
                const uint8_t bb = pos == P ? b : seq[pos];
                const int v = dev_base2val(bb);
                ok = ok && (v >= 0); code = (code << 2) | (v & 3); field |= ((bb >> 1) & 3) << (2 * k);
            }
            if (ok) {
                if (clean) atomicAdd(&D.kmer[side * FP_KMER_BINS + field], sg);
                else red_add64(&G[fp_off_kmer(&L, side * 2 + 1, code)], (unsigned long long)(long long)sg);
            }
        }
    }
}

/* t_patch_delta for a CLEAN row (bases in {A,C,G,T,N}, qualities < 128), word-sized: qualities and the per-cycle counters are two
 * signed updates each, the five 5-mers around P come from ONE pass over the nine bytes P-4 .. P+4 (2-bit codes + validity), read
 * while seq[P] still holds the old base. */
__device__ __noinline__ void t_patch_delta_clean(const DeltaAcc D, int side, const uint8_t* seq, int l0, int P, uint8_t ob, uint8_t oq, uint8_t nb, uint8_t nq) {
    FP_SMEM(D.cyc);    FP_SMEM(D.kmer);    FP_SMEM(D.qh);    FP_SMEM(seq);
    atomicAdd(&D.qh[side * FP_QUAL_BINS + oq], -1);
    atomicAdd(&D.qh[side * FP_QUAL_BINS + nq], +1);
    if (P < D.cycles) {
        int* c0 = D.cyc + side * D.cycles * 20 + P * 20;
        int* co = c0 + ((0x43F21F0Fu >> (4 * (ob & 7))) & 0xF) * 4;            /* base&7: A1 C3 T4 N6 G7 -> bin 0..4 */
        int* cn = c0 + ((0x43F21F0Fu >> (4 * (nb & 7))) & 0xF) * 4;
        atomicAdd(&co[0], -1); atomicAdd(&cn[0], +1);
        if (oq >= '5') atomicAdd(&co[1], -1);
        if (nq >= '5') atomicAdd(&cn[1], +1);
        if (oq >= '?') atomicAdd(&co[2], -1);
        if (nq >= '?') atomicAdd(&cn[2], +1);
        atomicAdd(&co[3], 33 - (int)oq); atomicAdd(&cn[3], (int)nq - 33);
    }
    uint32_t Z = 0, V = 0;                                                     /* digit k = position P-4+k */
    #pragma unroll
    for (int k = 0; k < 9; k++) {
        const int pos = P - 4 + k;
        const bool inb = pos >= 0 && pos < l0;
        const uint32_t bb = inb ? seq[pos] : (uint32_t)'N';
        Z |= ((bb >> 1) & 3u) << (2 * k);
        V |= (bb != (uint32_t)'N' ? 1u : 0u) << k;
    }
    const uint32_t Zn = (Z & ~(3u << 8)) | ((((uint32_t)nb >> 1) & 3u) << 8), Vn = (V & ~16u) | (nb != 'N' ? 16u : 0u);
    int* km = D.kmer + side * FP_KMER_BINS;
    #pragma unroll
    for (int w = 0; w < 5; w++) {                                              /* window ending at P+w = digits w .. w+4 */
        if (((V >> w) & 31u) == 31u) atomicAdd(&km[(Z >> (2 * w)) & 0x3FFu], -1);
        if (((Vn >> w) & 31u) == 31u) atomicAdd(&km[(Zn >> (2 * w)) & 0x3FFu], +1);
    }
}

/* complement of a base of a clean row (util.h:16-33 restricted to A,C,G,T,N): table indexed by base & 7 */
__device__ __forceinline__ uint8_t comp_clean(uint8_t b) {
    /* index 1 'A'->'T'  3 'C'->'G'  4 'T'->'A'  6 'N'->'N'  7 'G'->'C' */
    const unsigned long long tab = 0x434E4E41474E544Eull;
    return (uint8_t)(tab >> (8 * (b & 7)));
}

/* ------------------------------------------------------------------------------------------------
 * BaseCorrector::correctByOverlapAnalysis  (basecorrector.cpp:21-83).  Positions are independent: a mismatching position is
 * rewritten at most once, from the bytes and qualities of that position alone.  Two lanes of the pair's group share the work by
 * DIRECTION: lane 0 applies "read 1 is right" (rewrites read 2, :42-50), lane 1 "read 2 is right" (rewrites read 1, :51-59) -- each
 * read is then changed by one lane only, in increasing position, so its statistics deltas telescope exactly; the two conditions
 * exclude each other on the original qualities and a rewritten position satisfies neither, so the lanes cannot disturb one another.
 * Writes the shared-memory rows, the HBM rows, the patch list and (clean rows) the bit planes.  Returns (via flags) which reads changed.
 * ------------------------------------------------------------------------------------------------ */
__device__ __forceinline__ void t_plane_set_base(uint32_t* pl, int PW, int pos, uint8_t base, uint8_t q) {
    const int w = pos >> 5; const uint32_t m = 1u << (pos & 31);
    const int c2 = (base >> 1) & 3; const bool n = (base == 'N');
    pl[w] = (pl[w] & ~m) | ((!n && (c2 & 1)) ? m : 0u);
    pl[PW + w] = (pl[PW + w] & ~m) | ((!n && (c2 & 2)) ? m : 0u);
    pl[2 * PW + w] = (pl[2 * PW + w] & ~m) | (n ? m : 0u);
    pl[3 * PW + w] = (pl[3 * PW + w] & ~m) | ((q < (uint8_t)c_p.qualified_qual) ? m : 0u);
}

__device__ __noinline__ int t_correct(const TRead r1, const TRead r2, uint32_t* pl1, uint32_t* pl2, int PW, const fp_ov_result ov,
                                      uint8_t* g1s, uint8_t* g1q, uint8_t* g2s, uint8_t* g2q, unsigned int pair_index, const PatchSink sink,
                                      BlockCounters* bc, const DeltaAcc D, unsigned long long* G, int l1, int l2, int role) {
    FP_SMEM(r1.seq());    FP_SMEM(r1.qual());    FP_SMEM(r2.seq());    FP_SMEM(r2.qual());    FP_SMEM(pl1);    FP_SMEM(pl2);    FP_SMEM(bc);    FP_SMEM(D.cyc);    FP_SMEM(D.kmer);    FP_SMEM(D.qh);
    /* role 0: rewrite read 2 where read 1 is right; role 1: rewrite read 1 where read 2 is right.  Returns the number of bases this lane rewrote. */
    if (ov.diff == 0 || !ov.overlapped) return 0;                           /* :23-24 */
    const int ol = ov.overlap_len;
    const int start1 = max(0, (int)ov.offset);
    const int start2 = r2.len - max(0, -(int)ov.offset) - 1;
    uint8_t* s1 = r1.seq() + r1.front; uint8_t* q1p = r1.qual() + r1.front;
    uint8_t* s2 = r2.seq() + r2.front; uint8_t* q2p = r2.qual() + r2.front;
    const signed char GOOD = 33 + 30, BAD = 33 + 14;
    int corrected = 0;
    const bool use_planes = r1.clean && r2.clean;
    const int e = r2.front + r2.len - 1, jb = r2.len - 1 - start2;          /* rc(r2) index of overlap position 0 */
    #pragma unroll 1
    for (int k = 0; k * 32 < ol; k++) {
        /* positions of this 32-chunk whose bases differ: from the planes (clean rows) or all of them (the byte test below decides) */
        uint32_t todo = low_mask(ol - 32 * k);
        if (use_planes) {
            const int s0 = e - (jb + 32 * k) - 31, abit = r1.front + start1 + 32 * k;
            const uint32_t rn = __brev(tp_bits_z(pl2 + 2 * PW, s0));
            const uint32_t rl_ = __brev(tp_bits_z(pl2, s0)), rh = ~__brev(tp_bits_z(pl2 + PW, s0)) & ~rn;
            todo &= (tp_bits(pl1, abit) ^ rl_) | (tp_bits(pl1 + PW, abit) ^ rh) | (tp_bits(pl1 + 2 * PW, abit) ^ rn);
        }
        #pragma unroll 1
        while (todo) {
            const int i = 32 * k + __ffs(todo) - 1;
            todo &= todo - 1;
            const int p1 = start1 + i, p2 = start2 - i;
            const signed char q1 = (signed char)q1p[p1], q2 = (signed char)q2p[p2];
            if (role == 0 ? !(q1 >= GOOD && q2 <= BAD) : !(q2 >= GOOD && q1 <= BAD)) continue;
            const uint8_t b1 = s1[p1], b2 = s2[p2];
            if (b1 == (use_planes ? comp_clean(b2) : dev_complement(b2))) continue;
            if (role == 0) {                                                   /* use R1 :42-50 */
                const uint8_t nb = use_planes ? comp_clean(b1) : dev_complement(b1);
                if (r2.clean) t_patch_delta_clean(D, 1, r2.seq(), l2, r2.front + p2, b2, (uint8_t)q2, nb, (uint8_t)q1);
                else t_patch_delta(D, G, false, 1, r2.seq(), l2, r2.front + p2, b2, (uint8_t)q2, nb, (uint8_t)q1);
                s2[p2] = nb; q2p[p2] = (uint8_t)q1; g2s[p2] = nb; g2q[p2] = (uint8_t)q1;
                if (r2.clean) t_plane_set_base(pl2, PW, r2.front + p2, nb, (uint8_t)q1);
                corrected++;
                atomicAdd(&bc->fr[FP_FR_CORRECTION + (nb & 7) * 9], 1u);       /* diagonal only, SURVEY App. A.6 */
                if (sink.count) {
                    const unsigned int slot = atomicAdd(sink.count, 1u);
                    if (slot < sink.cap) { fp_patch pt; pt.pair = pair_index; pt.pos = (uint16_t)(r2.front + p2); pt.which = 1; pt.base = nb; pt.qual = (uint8_t)q1; pt.old_base = b2; pt.old_qual = (uint8_t)q2; pt._pad = 0; sink.patches[slot] = pt; }
                }
            } else {                                                           /* use R2 :51-59 */
                const uint8_t nb = use_planes ? comp_clean(b2) : dev_complement(b2);
                if (r1.clean) t_patch_delta_clean(D, 0, r1.seq(), l1, r1.front + p1, b1, (uint8_t)q1, nb, (uint8_t)q2);
                else t_patch_delta(D, G, false, 0, r1.seq(), l1, r1.front + p1, b1, (uint8_t)q1, nb, (uint8_t)q2);
                s1[p1] = nb; q1p[p1] = (uint8_t)q2; g1s[p1] = nb; g1q[p1] = (uint8_t)q2;
                if (r1.clean) t_plane_set_base(pl1, PW, r1.front + p1, nb, (uint8_t)q2);
                corrected++;
                atomicAdd(&bc->fr[FP_FR_CORRECTION + (nb & 7) * 9], 1u);
                if (sink.count) {
                    const unsigned int slot = atomicAdd(sink.count, 1u);
                    if (slot < sink.cap) { fp_patch pt; pt.pair = pair_index; pt.pos = (uint16_t)(r1.front + p1); pt.which = 0; pt.base = nb; pt.qual = (uint8_t)q2; pt.old_base = b1; pt.old_qual = (uint8_t)q1; pt._pad = 0; sink.patches[slot] = pt; }
                }
            }
        }
    }
    return corrected;
}

/* ------------------------------------------------------------------------------------------------
 * Base correction, distributed form (clean pairs).  A pair with a 3' low-quality tail inside its overlap can have dozens of
 * correctable positions; one lane working through them holds back its whole warp -- and, behind the tile's barrier, the CTA.
 * So the pair's lanes only DECIDE (which mismatching positions are rewritten, from the two quality bytes) and put every
 * correction on the tile's work list; then ONE LANE PER CORRECTION (all warps of the CTA) does the statistics deltas, the
 * patch entry and, after a barrier, the rewrite.  Everything about one correction is independent of the others except the
 * 5-mer delta of corrections less than five bases apart on one read: each affected window (ending at x in [P, P+4]) is taken
 * by the LAST corrected position not beyond x (the per-row mask of corrected positions tells), with its old bases from the
 * still unmodified row and its new bases from the partner read (position y of the rewritten read faces c - y of the other).
 * entry = row | which << 7 | P << 8 | Pp << 18   (which = the read that is rewritten, P its row position, Pp the partner's)
 * ------------------------------------------------------------------------------------------------ */
#define FP_CORR_CAP 1024               /* corrections of one tile; more go the sequential way */
__device__ __noinline__ bool t_correct_decide(const TRead r1, const TRead r2, int PW, const fp_ov_result ov, int row, int sub, int g,
                                              uint32_t* list, int* nlist, int cap, uint32_t* cm1, uint32_t* cm2) {
    FP_SMEM(r1.qual());    FP_SMEM(r2.qual());    FP_SMEM(r1.pl());    FP_SMEM(r2.pl());    FP_SMEM(list);    FP_SMEM(nlist);    FP_SMEM(cm1);    FP_SMEM(cm2);
    bool overflow = false;
    const int ol = ov.overlap_len;
    const int start1 = max(0, (int)ov.offset);
    const int start2 = r2.len - max(0, -(int)ov.offset) - 1;
    const uint8_t* q1p = r1.qual() + r1.front; const uint8_t* q2p = r2.qual() + r2.front;
    const signed char GOOD = 33 + 30, BAD = 33 + 14;                          /* basecorrector.cpp:26-27 */
    const uint32_t *pl1 = r1.pl(), *pl2 = r2.pl();
    const int e = r2.front + r2.len - 1, jb = r2.len - 1 - start2;           /* rc(r2) index of overlap position 0 */
    /* mismatching positions of the overlap, 32 per word: lane `sub` of the group compares the words k = sub, sub + g, ... (three plane
       fields of each read per word) and the group passes them round by shuffle, instead of every lane comparing every word */
    const unsigned gm = group_mask(g);
    const int nw = (ol + 31) >> 5;
    uint32_t mine[2] = {0u, 0u};                                               /* 2 g = 8 words: a PE row has at most 256 bases (fp_ctx_create) */
    #pragma unroll
    for (int kk = 0; kk < 2; kk++) {
        const int k = sub + g * kk;
        if (k < nw) {
            const int s0 = e - (jb + 32 * k) - 31, abit = r1.front + start1 + 32 * k;
            const uint32_t rn = __brev(tp_bits_z(pl2 + 2 * PW, s0));
            const uint32_t rl_ = __brev(tp_bits_z(pl2, s0)), rh = ~__brev(tp_bits_z(pl2 + PW, s0)) & ~rn;
            mine[kk] = ((tp_bits(pl1, abit) ^ rl_) | (tp_bits(pl1 + PW, abit) ^ rh) | (tp_bits(pl1 + 2 * PW, abit) ^ rn)) & low_mask(ol - 32 * k);
        }
    }
    #pragma unroll 1
    for (int k = 0; k < nw; k++) {
        const int kk = k / g;
        const uint32_t w = kk == 0 ? mine[0] : mine[1];
        uint32_t todo = __shfl_sync(gm, w, (lane_id() & ~(g - 1)) + (k % g));
        /* a low-quality tail puts its mismatches side by side: the group's lanes take the positions i with i % g == sub, so one
           bad tail is shared by all of them */
        todo &= (g == 4 ? 0x11111111u : g == 2 ? 0x55555555u : 0xFFFFFFFFu) << sub;
        #pragma unroll 1
        while (todo) {
            const int i = 32 * k + __ffs(todo) - 1;
            todo &= todo - 1;
            const int p1 = start1 + i, p2 = start2 - i;
            const signed char q1 = (signed char)q1p[p1], q2 = (signed char)q2p[p2];
            int which;
            if (q1 >= GOOD && q2 <= BAD) which = 1;                            /* read 1 is right: rewrite read 2 (:42-50) */
            else if (q2 >= GOOD && q1 <= BAD) which = 0;                       /* read 2 is right: rewrite read 1 (:51-59) */
            else continue;
            const int P1 = r1.front + p1, P2 = r2.front + p2;
            const int slot = atomicAdd(nlist, 1);
            if (slot >= cap) { overflow = true; continue; }                    /* left to the sequential path after the distributed one */
            list[slot] = (uint32_t)row | ((uint32_t)which << 7) | ((uint32_t)(which ? P2 : P1) << 8) | ((uint32_t)(which ? P1 : P2) << 18);
            if (which) atomicOr(&cm2[P2 >> 5], 1u << (P2 & 31)); else atomicOr(&cm1[P1 >> 5], 1u << (P1 & 31));
        }
    }
    return overflow;
}

/* one correction: statistics deltas (post-filter), patch entry (unless the caller writes it: sink.count == nullptr), correction matrix.
   Rows are still unmodified.  Returns old base | old quality << 8 | new base << 16 | new quality << 24. */
__device__ __noinline__ uint32_t t_correct_item(uint32_t entry, const uint8_t* tile0, int tile_array_bytes, int S, int T, const uint16_t* s_len, const uint32_t* cm,
                                            int CMW, const DeltaAcc D, BlockCounters* bc, const PatchSink sink, unsigned int pair_index) {
    FP_SMEM(tile0);    FP_SMEM(s_len);    FP_SMEM(cm);    FP_SMEM(D.cyc);    FP_SMEM(D.kmer);    FP_SMEM(D.qh);    FP_SMEM(bc);
    const int row = entry & 0x7F, which = (entry >> 7) & 1, P = (entry >> 8) & 0x3FF, Pp = (entry >> 18) & 0x3FF;
    const uint8_t* mseq = tile0 + (which * 2) * tile_array_bytes + row * S; const uint8_t* mqual = mseq + tile_array_bytes;
    const uint8_t* pseq = tile0 + ((which ^ 1) * 2) * tile_array_bytes + row * S; const uint8_t* pqual = pseq + tile_array_bytes;
    const uint32_t* mcm = cm + (which * T + row) * CMW;
    const int l0 = s_len[which * T + row], c = P + Pp;
    const uint8_t ob = mseq[P], oq = mqual[P], nb = comp_clean(pseq[Pp]), nq = pqual[Pp];
    const int side = which;
    atomicAdd(&D.qh[side * FP_QUAL_BINS + oq], -1);
    atomicAdd(&D.qh[side * FP_QUAL_BINS + nq], +1);
    if (P < D.cycles) {
        int* c0 = D.cyc + side * D.cycles * 20 + P * 20;
        int* co = c0 + ((0x43F21F0Fu >> (4 * (ob & 7))) & 0xF) * 4;            /* base&7: A1 C3 T4 N6 G7 -> bin 0..4 */
        int* cn = c0 + ((0x43F21F0Fu >> (4 * (nb & 7))) & 0xF) * 4;
        atomicAdd(&co[0], -1); atomicAdd(&cn[0], +1);
        if (oq >= '5') atomicAdd(&co[1], -1);
        if (nq >= '5') atomicAdd(&cn[1], +1);
        if (oq >= '?') atomicAdd(&co[2], -1);
        if (nq >= '?') atomicAdd(&cn[2], +1);
        atomicAdd(&co[3], 33 - (int)oq); atomicAdd(&cn[3], (int)nq - 33);
    }
    /* 5-mers: digit k = position P-4+k; old codes from the row, new codes with every corrected position of the window taken from the partner */
    uint32_t Z = 0, V = 0, Zn = 0, Vn = 0, CMB = 0;
    #pragma unroll
    for (int k = 0; k < 9; k++) {
        const int pos = P - 4 + k;
        const bool inb = pos >= 0 && pos < l0;
        const uint32_t bb = inb ? mseq[pos] : (uint32_t)'N';
        const bool corr = inb && ((mcm[pos >> 5] >> (pos & 31)) & 1u);
        const int pp = c - pos;
        const uint32_t nn_ = corr ? (uint32_t)comp_clean(pseq[pp]) : bb;       /* a corrected position faces a valid partner position */
        Z |= ((bb >> 1) & 3u) << (2 * k); V |= (bb != (uint32_t)'N' ? 1u : 0u) << k;
        Zn |= ((nn_ >> 1) & 3u) << (2 * k); Vn |= (nn_ != (uint32_t)'N' ? 1u : 0u) << k;
        CMB |= (corr ? 1u : 0u) << k;
    }
    int* km = D.kmer + side * FP_KMER_BINS;
    #pragma unroll
    for (int w = 0; w < 5; w++) {                                              /* window ending at P+w = digits w .. w+4; mine iff no corrected position in (P, P+w] */
        if ((CMB >> 5) & ((1u << w) - 1u)) continue;
        if (((V >> w) & 31u) == 31u) atomicAdd(&km[(Z >> (2 * w)) & 0x3FFu], -1);
        if (((Vn >> w) & 31u) == 31u) atomicAdd(&km[(Zn >> (2 * w)) & 0x3FFu], +1);
    }
    atomicAdd(&bc->fr[FP_FR_CORRECTION + (nb & 7) * 9], 1u);                   /* diagonal only, SURVEY App. A.6 */
    if (sink.count) {
        const unsigned int slot = atomicAdd(sink.count, 1u);
        if (slot < sink.cap) { fp_patch pt; pt.pair = pair_index; pt.pos = (uint16_t)P; pt.which = (uint8_t)which; pt.base = nb; pt.qual = nq; pt.old_base = ob; pt.old_qual = oq; pt._pad = 0; sink.patches[slot] = pt; }
    }
    return (uint32_t)ob | ((uint32_t)oq << 8) | ((uint32_t)nb << 16) | ((uint32_t)nq << 24);
}

/* the rewrite itself: shared-memory row, HBM row, bit planes (other lanes may touch the same plane words: atomics) */
__device__ __forceinline__ uint32_t t_correct_apply(uint32_t entry, uint8_t* tile0, int tile_array_bytes, int S, int T, uint32_t* planes, int PSTR, int PW,
                                                uint8_t* gseq, uint8_t* gqual) {
    const int row = entry & 0x7F, which = (entry >> 7) & 1, P = (entry >> 8) & 0x3FF, Pp = (entry >> 18) & 0x3FF;
    uint8_t* mseq = tile0 + (which * 2) * tile_array_bytes + row * S; uint8_t* mqual = mseq + tile_array_bytes;
    const uint8_t* pseq = tile0 + ((which ^ 1) * 2) * tile_array_bytes + row * S; const uint8_t* pqual = pseq + tile_array_bytes;
    const uint8_t nb = comp_clean(pseq[Pp]), nq = pqual[Pp];
    const uint32_t old = (uint32_t)mseq[P] | ((uint32_t)mqual[P] << 8);      /* returned: old base | old quality << 8 */
    mseq[P] = nb; mqual[P] = nq; gseq[P] = nb; gqual[P] = nq;
    uint32_t* pl = planes + (which * T + row) * PSTR + (P >> 5);
    const uint32_t m = 1u << (P & 31);
    const int c2 = (nb >> 1) & 3; const bool n = (nb == 'N');
    if (!n && (c2 & 1)) atomicOr(&pl[0], m); else atomicAnd(&pl[0], ~m);
    if (!n && (c2 & 2)) atomicOr(&pl[PW], m); else atomicAnd(&pl[PW], ~m);
    if (n) atomicOr(&pl[2 * PW], m); else atomicAnd(&pl[2 * PW], ~m);
    if (nq < (uint8_t)c_p.qualified_qual) atomicOr(&pl[3 * PW], m); else atomicAnd(&pl[3 * PW], ~m);
    return old;
}

/* ------------------------------------------------------------------------------------------------
 * AdapterTrimmer::trimBySequence  (adaptertrimmer.cpp:64-157), one thread per read.
 * Scan 1 on planes (clean read + clean adapter) or bytes; scans 2/3 in the closed form of dev_gap_scan,
 * evaluated sequentially (O(alen)).
 * ------------------------------------------------------------------------------------------------ */
__device__ __forceinline__ int t_gap_scan(const uint8_t* ins, const uint8_t* norm, int cmax, int cmin) {
    /* largest c in [cmin,cmax] with min_{1<=i<=c-1}(P1[i]-P2[i]) + P2[c] <= c/8 - 1, else -1 (see dev_gap_scan) */
    if (cmax < cmin || cmax < 2) return -1;
    int p1 = 0, p2 = 0, runmin = 1 << 20, best = -1;
    for (int j = 0; j < cmax; j++) {
        /* here p1 = P1[j], p2 = P2[j]; M[j+1] = runmin = min_{1<=i<=j} */
        const int c = j + 1;                                               /* evaluate c = j+1 needs M[c] (i<=c-1=j) and P2[c] */
        p1 += (ins[j] != norm[j]);
        const int p2n = p2 + (ins[j + 1] != norm[j]);                      /* P2[j+1] */
        if (c >= 2 && c >= cmin && runmin + p2n <= c / 8 - 1) best = c;
        /* extend runmin with i = j+1: P1[j+1] - P2[j+1] */
        runmin = min(runmin, p1 - p2n);
        p2 = p2n;
    }
    return best;
}

/* can the one-gap scan over lengths <= cmax accept anything?  D1 / D2: aligned / shifted mismatch bits (bit j = position j).
 * A length c in [8k, 8k+7] is accepted only if some split i has (aligned mismatches before i) + (shifted mismatches from i to c) <= k - 1;
 * the same quantity over the first K = 8k positions only, B_K = min_i popc(D1 & low(i)) + popc(D2 & low(K) & ~low(i)), is a lower bound for
 * every c >= K and grows with K.  So: some k with B_8k <= k - 1 must exist, and once B_K exceeds the largest allowance nothing longer can hit.
 * Random sequence fails at K = 8 nine times out of ten; what passes there is checked at 16, 24, 32 ... before the byte scan is paid. */
__device__ __noinline__ bool gap_may_hit(unsigned long long D1, unsigned long long D2, int cmax) {
    const int amax = cmax / 8 - 1;                                        /* c/8 - 1 < 0 for every c < 8 */
    const int kmax = min(cmax, 64) >> 3;
    /* B_K = popc(D2 & low(K)) + min_{0<=i<=K} S(i),  S(i) = popc(D1 & low(i)) - popc(D2 & low(i)): one walk over the bits, checked every 8 */
    int S = 0, M = 0, c2 = 0;
    #pragma unroll 1
    for (int k = 1; k <= kmax; k++) {
        const uint32_t b1 = (uint32_t)D1 & 0xFFu, b2 = (uint32_t)D2 & 0xFFu;
        D1 >>= 8; D2 >>= 8;
        c2 += __popc(b2);
        #pragma unroll
        for (int i = 0; i < 8; i++) { S += (int)((b1 >> i) & 1u) - (int)((b2 >> i) & 1u); M = min(M, S); }
        const int v = c2 + M;
        if (v <= k - 1) return true;
        if (v > amax) return false;
    }
    return false;
}

/* result of an adapter trimmer: 0 = not trimmed, else at_pack(new length, adapter position, adapter bases) -- one register
   instead of reference outputs, so the caller's read state need not have an address */
__device__ __forceinline__ unsigned long long at_pack(int len, int pos, int bases) {
    return 1ull << 63 | (unsigned long long)(uint32_t)len | (unsigned long long)(uint16_t)(int16_t)pos << 32 | (unsigned long long)(uint32_t)bases << 48;
}
__device__ __forceinline__ int at_len(unsigned long long t) { return (int)(uint32_t)t; }
__device__ __forceinline__ int at_pos(unsigned long long t) { return (int)(int16_t)(uint16_t)(t >> 32); }
__device__ __forceinline__ int at_bases(unsigned long long t) { return (int)((t >> 48) & 0x7FFFu); }

__device__ __noinline__ unsigned long long t_trim_by_sequence(const TRead r, const uint8_t* adata, int alen, int matchReq, int aidx, int PW,
                                                              BlockCounters* bc, int sub, int g, const EventSink ev, unsigned int unit, int which) {
    FP_SMEM(r.seq());    FP_SMEM(r.pl());    FP_SMEM(bc);
    const int rlen = r.len;
    const uint8_t* rdata = r.seq() + r.front;
    if (alen < matchReq) return 0ull;                                     /* :73-74 */
    int start = 0;
    if (alen >= 16) start = -4; else if (alen >= 12) start = -3; else if (alen >= 8) start = -2;
    bool found = false;
    int pos = 0;
    const bool planes = r.clean && c_p.adapter_clean[aidx];
    /* 64-bit plane fields of the read start and of the adapter (adapters up to 64 bases): the negative starts of scan 1 and the
       quick rejects of scans 2 / 3 are popcounts on them */
    const bool planes64 = planes && alen <= 64;
    unsigned long long R_lo = 0, R_hi = 0, R_nn = 0, A_lo = 0, A_hi = 0, A_nn = 0;
    if (planes64) {
        const uint32_t* ap = c_p.adapter_planes + aidx * 24;
        A_lo = (unsigned long long)__ldg(ap) | ((unsigned long long)__ldg(ap + 1) << 32);
        A_hi = (unsigned long long)__ldg(ap + 8) | ((unsigned long long)__ldg(ap + 9) << 32);
        A_nn = (unsigned long long)__ldg(ap + 16) | ((unsigned long long)__ldg(ap + 17) << 32);
        const unsigned long long live = mask64(rlen);
        R_lo = tp_bits64(r.pl(), r.front) & live; R_hi = tp_bits64(r.pl() + PW, r.front) & live; R_nn = tp_bits64(r.pl() + 2 * PW, r.front) & live;
    }
    /* scan 1 (:87-100) */
    for (int p = start; p < 0 && p < rlen - matchReq && !found; p++) {
        const int cmplen = min(rlen - p, alen), so = -p, n = cmplen - so;
        int mm = 0;
        if (planes64) mm = __popcll(((R_lo ^ (A_lo >> so)) | (R_hi ^ (A_hi >> so)) | (R_nn ^ (A_nn >> so))) & mask64(n));
        else for (int k = 0; k < n; k++) mm += (adata[so + k] != rdata[k]);
        if (mm <= cmplen / 8) { found = true; pos = p; }
    }
    if (!found) {
        const int npos = rlen - matchReq;
        int my_p = 1 << 20;
        if (planes) {
            const uint32_t* alo = c_p.adapter_planes + aidx * 24; const uint32_t* ahi = alo + 8; const uint32_t* ann = alo + 16;
            const uint32_t *plo = r.pl(), *phi = r.pl() + PW, *pnn = r.pl() + 2 * PW;
            const int nw = (alen + 31) >> 5;
            auto full_check = [&](int p) -> bool {                         /* exact count over the whole compared length */
                const int cmplen = min(rlen - p, alen);
                int mm = 0;
                for (int k = 0; k < nw && 32 * k < cmplen; k++) {
                    const int bit = r.front + p + 32 * k;
                    const uint32_t x = (tp_bits(plo, bit) ^ __ldg(alo + k)) | (tp_bits(phi, bit) ^ __ldg(ahi + k)) | (tp_bits(pnn, bit) ^ __ldg(ann + k));
                    mm += __popc(x & low_mask(cmplen - 32 * k));
                }
                return mm <= cmplen / 8;
            };
            /* main range: the first a0 = min(alen,32) adapter bases lie inside the read.  Same one-plane word filter as the overlap scan
               (t_ov_word_hits on X = lo ^ hi: bases whose X bits differ are different bases; allowance alen/8 bounds every position's own):
               a lane takes a whole plane word = 32 consecutive positions, branch-free; survivors get the exact three-plane count. */
            const int a0 = min(alen, 32);
            const int pmain = min(npos, rlen - a0 + 1);
            const uint32_t M0 = low_mask(a0), A_lo = __ldg(alo), A_hi = __ldg(ahi), A_nn = __ldg(ann);
            const int amax = alen / 8;
            if (pmain > 0) {
                const uint32_t AX = (A_lo ^ A_hi) & M0;
                const int blo = r.front, bhi = r.front + pmain - 1;
                #pragma unroll 1
                for (int w = (blo >> 5) + sub; w <= (bhi >> 5) && my_p == (1 << 20); w += g) {
                    const uint32_t W0 = plo[w] ^ phi[w], W1 = plo[w + 1] ^ phi[w + 1];
                    uint32_t hits = t_ov_word_hits(W0, W1, AX, M0, amax + 1);
                    hits &= low_mask(bhi - 32 * w + 1) & ~low_mask(blo - 32 * w);
                    while (hits) {
                        const int sh = __ffs(hits) - 1;
                        hits &= hits - 1;
                        const int p = 32 * w + sh - r.front;
                        if (full_check(p)) { my_p = p; break; }
                    }
                }
            }
            /* tail: the adapter runs past the read end, position p compares the read's last c = rlen - p bases with the adapter's first c.
               The read's last 32 bases are one constant field per plane; c goes down as p goes up. */
            if (group_min(my_p, g) == (1 << 20) && npos > pmain) {
                const int tb = r.front + rlen - 32;
                const uint32_t T_lo = tp_bits_z(plo, tb), T_hi = tp_bits_z(phi, tb), T_nn = tp_bits_z(pnn, tb);
                #pragma unroll 1
                for (int pp = max(pmain, 0) + sub; pp < npos; pp += g) {
                    const int c = rlen - pp;                               /* matchReq < c < a0 <= 32 */
                    const uint32_t x = (((T_lo >> (32 - c)) ^ A_lo) | ((T_hi >> (32 - c)) ^ A_hi) | ((T_nn >> (32 - c)) ^ A_nn)) & low_mask(c);
                    if (__popc(x) <= c / 8) { my_p = pp; break; }
                }
            }
        } else {
            for (int p = sub; p < npos; p += g) {
                const int cmplen = min(rlen - p, alen), allowed = cmplen / 8;
                int mm = 0;
                for (int k = 0; k < cmplen && mm <= allowed; k++) mm += (adata[k] != rdata[p + k]);
                if (mm <= allowed) { my_p = p; break; }
            }
        }
        const int best = group_min(my_p, g);
        if (best < (1 << 20)) { found = true; pos = best; }
    }
    /* Scans 2 / 3 accept a length c only if some split i has (aligned mismatches before i) + (shifted mismatches from i to c)
       <= c/8 - 1, which is negative below c = 8 and at most cmax/8 - 1 overall; the same quantity restricted to the first 8
       positions is a lower bound for every c >= 8, so when even that exceeds the largest allowance the scan cannot hit. */
    const unsigned long long D1 = (R_lo ^ A_lo) | (R_hi ^ A_hi) | (R_nn ^ A_nn);                                  /* read[j] != adapter[j] */
    const int cmax2 = min(rlen - 1, alen), cmax3 = min(rlen, alen - 1);
    bool may2 = true, may3 = true;
    if (planes64 && !found && rlen - matchReq > 0) {
        /* both quick rejects at once: even lanes of the group test scan 2 (read[j+1] != adapter[j]), odd lanes scan 3 (adapter[j+1] != read[j]) */
        const bool odd = (g >= 2) && (sub & 1);
        const unsigned long long D2 = odd ? (((A_lo >> 1) ^ R_lo) | ((A_hi >> 1) ^ R_hi) | ((A_nn >> 1) ^ R_nn))
                                          : (((R_lo >> 1) ^ A_lo) | ((R_hi >> 1) ^ A_hi) | ((R_nn >> 1) ^ A_nn));
        const bool m = gap_may_hit(D1, D2, odd ? cmax3 : cmax2);
        if (g >= 2) {
            const unsigned gm = group_mask(g);
            const int l0 = lane_id() & ~(g - 1);
            may2 = __shfl_sync(gm, (int)m, l0) != 0; may3 = __shfl_sync(gm, (int)m, l0 + 1) != 0;
        } else {
            may2 = m;
            may3 = gap_may_hit(D1, ((A_lo >> 1) ^ R_lo) | ((A_hi >> 1) ^ R_hi) | ((A_nn >> 1) ^ R_nn), cmax3);
        }
    }
    if (!found && rlen - matchReq - 1 > 0) {                              /* scan 2 (:105-118) */
        const int c = may2 ? t_gap_scan(rdata, adata, cmax2, matchReq + 1) : -1;
        if (c >= 0) { found = true; pos = (c == cmax2) ? 0 : rlen - 1 - c; }
    }
    if (!found && rlen - matchReq > 0) {                                  /* scan 3 (:122-135) */
        const int c = may3 ? t_gap_scan(adata, rdata, cmax3, matchReq + 1) : -1;
        if (c >= 0) { found = true; pos = (c == cmax3) ? 0 : rlen - c; }
    }
    if (found) {                                                          /* :137-154 */
        int abases, len = r.len;
        if (pos < 0) { abases = alen + pos; len = 0; }
        else { abases = rlen - pos; if (pos <= len) len = pos; }
        if (abases > 0 && sub == 0) {
            atomicAdd(&bc->fr[FP_FR_ADAPTER_BASES], (unsigned)abases);
            /* the string FilterResult::addAdapterTrimmed histograms (:139-152): a prefix of the adapter, or the read's tail */
            const int key = (aidx < 2 ? 0 : 2048) + which * 1024 + (aidx < 2 ? 0 : aidx - 2);
            if (pos < 0) push_event(ev, unit, which, FP_EV_ADAPTER, key, 0, abases, aidx);
            else push_event(ev, unit, which, FP_EV_READ, key, r.front + pos, abases, aidx);
        }
        return at_pack(len, pos, max(abases, 0));
    }
    return 0ull;
}

/* AdapterTrimmer::trimByMultiSequences (adaptertrimmer.cpp:48-62): applies every hit to r (length, adapter position, adapter
   bases added to *bases); returns whether any adapter trimmed */
__device__ __forceinline__ bool t_trim_by_multi(TRead& r, int PW, int& pos, int& bases, BlockCounters* bc, int sub, int g, const EventSink ev, unsigned int unit, int which) {
    bool trimmed = false;
    for (int i = 0; i < c_p.n_fasta; i++) {
        const unsigned long long t = t_trim_by_sequence(r, c_p.adapters + c_p.fasta_off[i], c_p.fasta_len[i], c_p.fasta_match_req, 2 + i, PW, bc, sub, g, ev, unit, which);
        if (t) { r.len = at_len(t); pos = at_pos(t); bases += at_bases(t); trimmed = true; }
    }
    return trimmed;
}

/* ------------------------------------------------------------------------------------------------
 * Filter::passFilter  (filter.cpp:15-57), one thread per read: planes for clean rows, bytes otherwise.
 * ------------------------------------------------------------------------------------------------ */
__device__ __noinline__ int t_pass_filter(const TRead r, int PW, const int16_t* lut) {
    FP_SMEM(r.pl());    FP_SMEM(r.seq());    FP_SMEM(r.qual());    FP_SMEM(lut);
    if (r.null || r.len == 0) return FP_FAIL_LENGTH;
    const int rlen = r.len;
    int lowq = 0, nb = 0, adj = 0;
    if (r.clean) {
        const uint32_t *plo = r.pl(), *phi = r.pl() + PW, *pnn = r.pl() + 2 * PW, *plq = r.pl() + 3 * PW;
        for (int k = 0; k * 32 < rlen; k++) {
            const int bit = r.front + 32 * k;
            const uint32_t m = low_mask(rlen - 32 * k);
            const uint32_t nn = tp_bits(pnn, bit);
            lowq += __popc(tp_bits(plq, bit) & m);
            nb += __popc(nn & m);
            if (c_p.complexity_filter) {
                const uint32_t d = (tp_bits(plo, bit) ^ tp_bits(plo, bit + 1)) | (tp_bits(phi, bit) ^ tp_bits(phi, bit + 1)) | (nn ^ tp_bits(pnn, bit + 1));
                adj += __popc(d & low_mask(rlen - 1 - 32 * k));
            }
        }
    } else {
        const uint8_t* s = r.seq() + r.front; const uint8_t* q = r.qual() + r.front;
        const uint8_t qq = (uint8_t)c_p.qualified_qual;
        for (int i = 0; i < rlen; i++) {
            lowq += (q[i] < qq); nb += (s[i] == 'N');
            if (i + 1 < rlen) adj += (s[i] != s[i + 1]);
        }
    }
    if (c_p.qual_filter) {
        if (lowq > (int)lut[(c_p.stride + 2) + rlen]) return FP_FAIL_QUALITY;
        if (c_p.avg_qual_req > 0) {
            const uint8_t* q = r.qual() + r.front;
            int tq = 0;
            for (int i = 0; i < rlen; i++) tq += (int)q[i] - 33;
            if ((tq / rlen) < c_p.avg_qual_req) return FP_FAIL_QUALITY;
        }
        if (nb > c_p.n_base_limit) return FP_FAIL_N_BASE;
    }
    if (c_p.length_filter) {
        if (rlen < c_p.length_required) return FP_FAIL_LENGTH;
        if (c_p.length_limit > 0 && rlen > c_p.length_limit) return FP_FAIL_TOO_LONG;
    }
    if (c_p.complexity_filter) {
        if (rlen <= 1) return FP_FAIL_COMPLEXITY;
        if (adj < (int)lut[2 * (c_p.stride + 2) + rlen]) return FP_FAIL_COMPLEXITY;
    }
    return FP_PASS_FILTER;
}

/* Filter::passFilter shared by the lanes of a group: lane `half` (0 / 1) of a lane PAIR counts the plane words k = half, half + 2, ...
 * of the pair's read, the two partial counts meet by one shuffle and both lanes hold the verdict.  PE groups give lanes 0, 1 to read 1
 * and lanes 2, 3 to read 2 (the caller exchanges the verdicts); every lane of the group must call. */
__device__ __noinline__ int t_pass_filter_pair(const TRead r, int PW, const int16_t* lut, int half, unsigned gm) {
    FP_SMEM(r.pl());    FP_SMEM(r.seq());    FP_SMEM(r.qual());    FP_SMEM(lut);
    const int rlen = (r.null || r.len == 0) ? 0 : r.len;
    int lowq = 0, nb = 0, adj = 0;
    if (r.clean) {
        const uint32_t *plo = r.pl(), *phi = r.pl() + PW, *pnn = r.pl() + 2 * PW, *plq = r.pl() + 3 * PW;
        for (int k = half; k * 32 < rlen; k += 2) {
            const int bit = r.front + 32 * k;
            const uint32_t m = low_mask(rlen - 32 * k);
            const uint32_t nn = tp_bits(pnn, bit);
            lowq += __popc(tp_bits(plq, bit) & m);
            nb += __popc(nn & m);
            if (c_p.complexity_filter) {
                const uint32_t d = (tp_bits(plo, bit) ^ tp_bits(plo, bit + 1)) | (tp_bits(phi, bit) ^ tp_bits(phi, bit + 1)) | (nn ^ tp_bits(pnn, bit + 1));
                adj += __popc(d & low_mask(rlen - 1 - 32 * k));
            }
        }
    } else if (half == 0) {
        const uint8_t* s = r.seq() + r.front; const uint8_t* q = r.qual() + r.front;
        const uint8_t qq = (uint8_t)c_p.qualified_qual;
        for (int i = 0; i < rlen; i++) {
            lowq += (q[i] < qq); nb += (s[i] == 'N');
            if (i + 1 < rlen) adj += (s[i] != s[i + 1]);
        }
    }
    int packed = lowq | (nb << 10) | (adj << 20);                          /* each count <= 1023 (row length) */
    packed += __shfl_xor_sync(gm, packed, 1);
    lowq = packed & 1023; nb = (packed >> 10) & 1023; adj = packed >> 20;
    if (rlen == 0) return FP_FAIL_LENGTH;
    if (c_p.qual_filter) {
        if (lowq > (int)lut[(c_p.stride + 2) + rlen]) return FP_FAIL_QUALITY;
        if (c_p.avg_qual_req > 0) {
            const uint8_t* q = r.qual() + r.front;
            int tq = 0;
            for (int i = 0; i < rlen; i++) tq += (int)q[i] - 33;
            if ((tq / rlen) < c_p.avg_qual_req) return FP_FAIL_QUALITY;
        }
        if (nb > c_p.n_base_limit) return FP_FAIL_N_BASE;
    }
    if (c_p.length_filter) {
        if (rlen < c_p.length_required) return FP_FAIL_LENGTH;
        if (c_p.length_limit > 0 && rlen > c_p.length_limit) return FP_FAIL_TOO_LONG;
    }
    if (c_p.complexity_filter) {
        if (rlen <= 1) return FP_FAIL_COMPLEXITY;
        if (adj < (int)lut[2 * (c_p.stride + 2) + rlen]) return FP_FAIL_COMPLEXITY;
    }
    return FP_PASS_FILTER;
}

/* ------------------------------------------------------------------------------------------------
 * --merge (peprocessor.cpp:519-560).  The merged read is never materialised: it is a view over the two tile rows
 * (OverlapAnalysis::merge, overlapanalysis.cpp:148-179): positions [0, n1) are s1[0, n1) (read 1 from its trimmed start), position
 * n1 + k is the complement of s2[n2 - 1 - k] with that base's quality (read 2 from its trimmed start).  n2 = 0: a plain read (the
 * unmerged reads of --include_unmerged).  A feature path, not a tuned one: the group's lanes share the positions, the Stats go to
 * the global block by RED (a merged read can be two rows long, longer than the block-private accumulators).
 * ------------------------------------------------------------------------------------------------ */
struct MView { const uint8_t *s1, *q1, *s2, *q2; int n1, n2; };
__device__ __forceinline__ uint8_t mv_base(const MView& v, int j) { return j < v.n1 ? v.s1[j] : dev_complement(v.s2[v.n2 - 1 - (j - v.n1)]); }
__device__ __forceinline__ uint8_t mv_qual(const MView& v, int j) { return j < v.n1 ? v.q1[j] : v.q2[v.n2 - 1 - (j - v.n1)]; }
__device__ __forceinline__ int group_sum(int v, int g) {
    const unsigned gm = group_mask(g);
    for (int o = g >> 1; o > 0; o >>= 1) v += __shfl_xor_sync(gm, v, o);
    return v;
}

/* Filter::passFilter (filter.cpp:15-57) of a view */
__device__ __noinline__ int t_pass_filter_view(const MView v, int sub, int g) {
    const int rlen = v.n1 + v.n2;
    if (rlen == 0) return FP_FAIL_LENGTH;
    int lowq = 0, nb = 0, tq = 0, adj = 0;
    const uint8_t qq = (uint8_t)c_p.qualified_qual;
    for (int i = sub; i < rlen; i += g) {
        const uint8_t b = mv_base(v, i), q = mv_qual(v, i);
        lowq += (q < qq); nb += (b == 'N'); tq += (int)q - 33;
        if (i + 1 < rlen) adj += (b != mv_base(v, i + 1));
    }
    lowq = group_sum(lowq, g); nb = group_sum(nb, g); tq = group_sum(tq, g); adj = group_sum(adj, g);
    if (c_p.qual_filter) {
        if (lowq > (int)c_p.lut_lowq[rlen]) return FP_FAIL_QUALITY;
        if (c_p.avg_qual_req > 0 && (tq / rlen) < c_p.avg_qual_req) return FP_FAIL_QUALITY;
        if (nb > c_p.n_base_limit) return FP_FAIL_N_BASE;
    }
    if (c_p.length_filter) {
        if (rlen < c_p.length_required) return FP_FAIL_LENGTH;
        if (c_p.length_limit > 0 && rlen > c_p.length_limit) return FP_FAIL_TOO_LONG;
    }
    if (c_p.complexity_filter) {
        if (rlen <= 1) return FP_FAIL_COMPLEXITY;
        if (adj < (int)c_p.lut_mindiff[rlen]) return FP_FAIL_COMPLEXITY;
    }
    return FP_PASS_FILTER;
}

/* Stats::statRead (stats.cpp:191-268, without the over-representation scan) of a view, into Stats `stats` of the global block */
__device__ __noinline__ void t_stat_view(unsigned long long* G, int stats, const MView v, int sub, int g) {
    const fp_counter_layout& L = c_p.L;
    const int rlen = v.n1 + v.n2;
    for (int i = sub; i < rlen; i += g) {
        const uint8_t base = mv_base(v, i), q = mv_qual(v, i);
        const int b = base & 7;
        if (q < FP_QUAL_BINS) red_add64(&G[fp_off_qualhist(&L, stats, q)], 1ull);
        if (i < L.cycles) {
            if (q >= '?') { red_add64(&G[fp_off_cycle(&L, stats, 0 * 8 + b, i)], 1ull); red_add64(&G[fp_off_cycle(&L, stats, 1 * 8 + b, i)], 1ull); }
            else if (q >= '5') red_add64(&G[fp_off_cycle(&L, stats, 1 * 8 + b, i)], 1ull);
            red_add64(&G[fp_off_cycle(&L, stats, 2 * 8 + b, i)], 1ull);
            red_add64(&G[fp_off_cycle(&L, stats, 3 * 8 + b, i)], (unsigned long long)(long long)((int)q - 33));
        }
        if (i >= 4) {
            int code = 0; bool ok = true;
            #pragma unroll
            for (int k = 0; k < 5; k++) { const int val = dev_base2val(mv_base(v, i - 4 + k)); ok = ok && (val >= 0); code = (code << 2) | (val & 3); }
            if (ok) red_add64(&G[fp_off_kmer(&L, stats, code)], 1ull);
        }
    }
}

__device__ __forceinline__ fp_read_result t_make_result(const TRead& r, int verdict, int pv, int flags, int apos, int abases, int pbase, int plen) {
    fp_read_result o;
    if (r.null) { o.front = 0; o.len = 0; flags |= FP_F_DROPPED; }
    else { o.front = (uint16_t)r.front; o.len = (uint16_t)r.len; }
    o.verdict = (uint8_t)verdict; o.flags = (uint8_t)flags; o.adapter_pos = (int16_t)apos; o.adapter_len = (uint16_t)abases;
    o.polyx_base = (uint8_t)pbase; o.pair_verdict = (uint8_t)pv; o.polyx_len = (uint16_t)plen; o.flags2 = 0;
    return o;
}
/* the record of a read whose unit the index filter removed (seprocessor.cpp:220-224, peprocessor.cpp:404-410) */
__device__ __forceinline__ fp_read_result t_index_filtered_result() {
    fp_read_result o;
    o.front = 0; o.len = 0; o.verdict = FP_FAIL_LENGTH; o.flags = FP_F_DROPPED; o.adapter_pos = 0; o.adapter_len = 0;
    o.polyx_base = 255; o.pair_verdict = FP_FAIL_LENGTH; o.polyx_len = 0; o.flags2 = FP_F2_INDEX_FILTERED;
    return o;
}

/* dense pass for TWO cycles (half a word column): acc[cyc 0..1][bin][kind] */
struct ColAcc2 { unsigned int v[2][NB][4]; };

/* table index used while counting (oldest base in the low digit, codes A0 C1 T2 G3) -> reference 5-mer index
   (oldest base in the high digit, base2val A0 T1 C2 G3; stats.cpp:248-266) */
__device__ __forceinline__ int kmer_ref_index(int f) {
    int r = 0;
    #pragma unroll
    for (int d = 0; d < 5; d++) {
        const int c = (f >> (2 * d)) & 3;
        r |= (((c & 1) << 1) | (c >> 1)) << (2 * (4 - d));
    }
    return r;
}

/* exact "byte is one of A,C,G,T" per byte (0/1 bytes): class by base&7 plus the upper-bit pattern */
__device__ __forceinline__ uint32_t exact_acgt(uint32_t w) {
    const uint32_t K = 0x01010101u;
    const uint32_t c0 = w & K, c1 = (w >> 1) & K, c2 = (w >> 2) & K, b3 = (w >> 3) & K, b4 = (w >> 4) & K;
    const uint32_t up = (~(w >> 5)) & (w >> 6) & (~(w >> 7)) & K;
    return ((c0 & (~c2 | c1) & ~b3 & ~b4) | (~c0 & ~c1 & c2 & ~b3 & b4)) & up;
}

/* dense pass, one step of 4 rows for a word that some of the rows do not fully cover (the read ends inside or before it).
 * Out of line on purpose: it is rare, and keeping it out of the hot loop keeps the 40 accumulators in registers there. */
__device__ __noinline__ void dense_masked_step(ColAcc2& acc, const uint8_t* ts, const uint8_t* tq, const uint16_t* lens, int r0, int S, int w4, int j0,
                                               unsigned sel, unsigned long long* G, int my_side) {
    FP_SMEM(ts); FP_SMEM(tq); FP_SMEM(lens);
    uint32_t xs[4], xq[4];
    #pragma unroll
    for (int kk = 0; kk < 4; kk++) {
        const int r = r0 + kk;
        const uint32_t m = window_mask(w4, 0, lens[r]);          /* rows beyond the tile have length 0 */
        uint32_t x = 0, q = 0;
        if (m) {
            const uint32_t K = 0x01010101u;
            x = *reinterpret_cast<const uint32_t*>(ts + r * S + w4) & m;
            q = *reinterpret_cast<const uint32_t*>(tq + r * S + w4) & m;
            /* bytes the register fast path cannot represent: base&7 in {0,2,5} or quality >= 128 -> exact global path */
            const uint32_t c0 = x & K, c1 = (x >> 1) & K, c2 = (x >> 2) & K;
            const uint32_t present = (m & K);
            uint32_t bad = present & (((~c0) & (~c2)) | (c0 & (~c1) & c2) | (q >> 7));
            if (bad) {
                #pragma unroll 1
                for (int j = j0; j < j0 + 2; j++)
                    if ((bad >> (8 * j)) & 1) {
                        const uint8_t bb = (uint8_t)(x >> (8 * j)), qb = (uint8_t)(q >> (8 * j));
                        slow_cycle_byte(G, my_side * 2, w4 + j, bb, qb);           /* dense feeds pre AND post */
                        slow_cycle_byte(G, my_side * 2 + 1, w4 + j, bb, qb);
                    }
                x &= ~(bad * 0xFFu);                                              /* drop them from the fast path */
            }
        }
        xs[kk] = x; xq[kk] = q;
    }
    const uint32_t t0 = __byte_perm(xs[0], xs[1], sel), t1 = __byte_perm(xs[2], xs[3], sel);
    const uint32_t u0 = __byte_perm(xq[0], xq[1], sel), u1 = __byte_perm(xq[2], xq[3], sel);
    acc_cycle(acc.v[0], __byte_perm(t0, t1, 0x5410), __byte_perm(u0, u1, 0x5410));
    acc_cycle(acc.v[1], __byte_perm(t0, t1, 0x7632), __byte_perm(u0, u1, 0x7632));
}

/* Dense column pass over one tile for one thread's two cycles (w4 + 2*my_half, +1) of one side: Stats::statRead's per-cycle
 * counters (stats.cpp:204-227), exact for any byte.  A function of its own so that the 40 accumulators get registers of their own
 * inside the hot loop whatever the rest of the kernel keeps live; between tiles they rest in the caller's frame and are loaded /
 * stored here ONCE per tile through the reference (by value they crossed local memory four times: 2 KB of L2 traffic per pair). */
__device__ __noinline__ void dense_tile(ColAcc2& acc_io, const uint8_t* ts, const uint8_t* tq, const uint16_t* lens, int rows, int S, int w4, int my_half,
                                           int rfirst, int rstep, unsigned long long* G, int my_side) {
    FP_SMEM(ts); FP_SMEM(tq); FP_SMEM(lens);
    unsigned int acc[2][NB][4];                      /* element-wise copies: the accumulators must live in registers in the loop */
    #pragma unroll
    for (int c = 0; c < 2; c++)
        #pragma unroll
        for (int b = 0; b < NB; b++)
            #pragma unroll
            for (int k = 0; k < 4; k++) acc[c][b][k] = acc_io.v[c][b][k];
    const int j0 = my_half * 2;
    const unsigned sel = my_half ? 0x7362u : 0x5140u;
    #pragma unroll (kDenseUnroll)
    for (int r0 = rfirst; r0 < rows; r0 += rstep) {
        /* rows beyond the tile have length 0, so the minimum also covers a partial tile */
        const uint2 l4 = *reinterpret_cast<const uint2*>(lens + r0);
        const uint32_t minl = min(min(l4.x & 0xFFFFu, l4.x >> 16), min(l4.y & 0xFFFFu, l4.y >> 16));
        const uint32_t maxl = max(max(l4.x & 0xFFFFu, l4.x >> 16), max(l4.y & 0xFFFFu, l4.y >> 16));
        const uint32_t cov = min(minl, (uint32_t)(w4 + 4));
        if ((uint32_t)w4 >= maxl) continue;           /* no row reaches this word */
        if (cov == min(maxl, (uint32_t)(w4 + 4))) {   /* the four rows cover the SAME bytes of this word: no masks, whole cycles in or out */
            uint32_t xs[4], xq[4];
            #pragma unroll
            for (int kk = 0; kk < 4; kk++) {
                xs[kk] = *reinterpret_cast<const uint32_t*>(ts + (r0 + kk) * S + w4);
                xq[kk] = *reinterpret_cast<const uint32_t*>(tq + (r0 + kk) * S + w4);
            }
            const uint32_t t0 = __byte_perm(xs[0], xs[1], sel), t1 = __byte_perm(xs[2], xs[3], sel);
            const uint32_t u0 = __byte_perm(xq[0], xq[1], sel), u1 = __byte_perm(xq[2], xq[3], sel);
            if ((uint32_t)(w4 + j0) < cov) acc_cycle_full(acc[0], __byte_perm(t0, t1, 0x5410), __byte_perm(u0, u1, 0x5410), G, my_side, w4 + j0);
            if ((uint32_t)(w4 + j0 + 1) < cov) acc_cycle_full(acc[1], __byte_perm(t0, t1, 0x7632), __byte_perm(u0, u1, 0x7632), G, my_side, w4 + j0 + 1);
            continue;
        }
        {   /* boundary words: rare, out of line; the accumulators travel through a copy so they stay in registers here */
            ColAcc2 tmp;
            #pragma unroll
            for (int c = 0; c < 2; c++)
                #pragma unroll
                for (int b = 0; b < NB; b++)
                    #pragma unroll
                    for (int k = 0; k < 4; k++) tmp.v[c][b][k] = acc[c][b][k];
            dense_masked_step(tmp, ts, tq, lens, r0, S, w4, j0, sel, G, my_side);
            #pragma unroll
            for (int c = 0; c < 2; c++)
                #pragma unroll
                for (int b = 0; b < NB; b++)
                    #pragma unroll
                    for (int k = 0; k < 4; k++) acc[c][b][k] = tmp.v[c][b][k];
        }
    }
    #pragma unroll
    for (int c = 0; c < 2; c++)
        #pragma unroll
        for (int b = 0; b < NB; b++)
            #pragma unroll
            for (int k = 0; k < 4; k++) acc_io.v[c][b][k] = acc[c][b][k];
}

/* ------------------------------------------------------------------------------------------------
 * Post-filter statistics of what the chain REMOVED from clean rows (failed reads, trimmed tails): the dense pass and the
 * histogram items credited every base of the tile to pre AND post, so the removed positions [lo, hi) of a row are taken out
 * of post again -- with the same machinery that counted them: a transposed dp4a pass over the removal list for the per-cycle
 * counters (dense_remove) and word-parallel histogram items for qualities and 5-mers (hist_remove_chunk), both into the
 * block-private signed accumulators.  One list per side; entry = row | lo << 8 | hi << 20; lists are zero-padded to a
 * multiple of four entries (hi = 0: nothing).
 * ------------------------------------------------------------------------------------------------ */
__device__ __forceinline__ uint32_t rm_pack(int row, int lo, int hi) { return (uint32_t)row | ((uint32_t)lo << 8) | ((uint32_t)hi << 20); }

/* The side's entries are kept in BUCKETS by lo >> 5 (bk: [nbk][bstride] entries, nb: their lengths): a removal [lo, hi) touches the word
 * column at w4 only if lo < w4 + 4, i.e. only if its bucket is <= (w4 + 3) >> 5 -- the column threads of the early cycles, where only
 * failed reads reach, skip the tail trims altogether.  The quads of four entries (buckets are zero-padded to quads) are dealt
 * round-robin to the `nsplit` threads of a column over all buckets together. */
__device__ __noinline__ void dense_remove(const uint32_t* bk, const int* nb, int nbk, int bstride, int part, int nsplit, const uint8_t* ts, const uint8_t* tq, int S, int w4, int my_half,
                                          int* dc, int cycles) {
    FP_SMEM(bk); FP_SMEM(nb); FP_SMEM(ts); FP_SMEM(tq); FP_SMEM(dc);
    unsigned int acc[2][NB][4];
    #pragma unroll
    for (int c = 0; c < 2; c++)
        #pragma unroll
        for (int b = 0; b < NB; b++)
            #pragma unroll
            for (int k = 0; k < 4; k++) acc[c][b][k] = 0;
    const int j0 = my_half * 2;
    const unsigned sel = my_half ? 0x7362u : 0x5140u;
    bool any = false;
    const int bmax = min(nbk - 1, (w4 + 3) >> 5);
    int qskip = part;                                 /* quads to pass over before my next one */
    #pragma unroll 1
    for (int b = 0; b <= bmax; b++) {
      const int nq = (nb[b] + 3) >> 2;
      const uint32_t* list = bk + b * bstride;
      int qi = qskip;
      #pragma unroll 1
      for (; qi < nq; qi += nsplit) {
        const uint4 e4 = *reinterpret_cast<const uint4*>(list + 4 * qi);
        const uint32_t es[4] = {e4.x, e4.y, e4.z, e4.w};
        uint32_t xs[4], xq[4], anym = 0;
        #pragma unroll
        for (int kk = 0; kk < 4; kk++) {
            const int row = es[kk] & 0xFF, lo = (es[kk] >> 8) & 0xFFF, hi = es[kk] >> 20;
            const uint32_t m = window_mask(w4, lo, hi);
            uint32_t x = 0, q = 0;
            if (m) {
                x = *reinterpret_cast<const uint32_t*>(ts + row * S + w4) & m;
                q = *reinterpret_cast<const uint32_t*>(tq + row * S + w4) & m;
            }
            xs[kk] = x; xq[kk] = q; anym |= m;
        }
        if (!anym) continue;
        any = true;
        const uint32_t t0 = __byte_perm(xs[0], xs[1], sel), t1 = __byte_perm(xs[2], xs[3], sel);
        const uint32_t u0 = __byte_perm(xq[0], xq[1], sel), u1 = __byte_perm(xq[2], xq[3], sel);
        acc_cycle(acc[0], __byte_perm(t0, t1, 0x5410), __byte_perm(u0, u1, 0x5410));
        acc_cycle(acc[1], __byte_perm(t0, t1, 0x7632), __byte_perm(u0, u1, 0x7632));
      }
      qskip = qi - nq;                                /* my next quad of the concatenation lies this far into the next bucket */
    }
    if (!any) return;
    #pragma unroll
    for (int c = 0; c < 2; c++) {
        const int cyc = w4 + j0 + c;
        if (cyc >= cycles) continue;
        #pragma unroll
        for (int b = 0; b < NB; b++) {
            const unsigned int nb = acc[c][b][0];
            if (nb == 0) continue;
            int* c4 = dc + (cyc * 5 + b) * 4;
            atomicAdd(&c4[0], -(int)nb);
            if (acc[c][b][1]) atomicAdd(&c4[1], -(int)acc[c][b][1]);
            if (acc[c][b][2]) atomicAdd(&c4[2], -(int)acc[c][b][2]);
            atomicAdd(&c4[3], -(int)(acc[c][b][3] - 33u * nb));
        }
    }
}

/* -1 in a block-private table at shared-window address `addr` iff bit `bit` of m is set */
#define smem_dec_bit(addr, m, bit) asm volatile("{ .reg .pred p; .reg .b32 t; and.b32 t, %1, %2; setp.ne.u32 p, t, 0; @p red.shared.add.u32 [%0], 0xffffffff; }" :: "r"(addr), "r"(m), "r"(1u << (bit)) : "memory")

/* qualities and 5-mers of the positions `rmask` of one 32-base chunk (chunk j of a clean row; sp / qp point at the chunk) out of the
 * post-filter histograms: qaddr / kaddr = shared-window addresses of this side's signed tables (kaddr 4 KB-aligned, indexed like the
 * pre-filter 5-mer table); nn_cur / nn_prev = N-plane words of this chunk and the one before it. */
__device__ __noinline__ void hist_remove_chunk(const uint8_t* sp, const uint8_t* qp, int j, uint32_t rmask, uint32_t nn_cur, uint32_t nn_prev,
                                               uint32_t qaddr, uint32_t kaddr, uint32_t kdummy) {
    FP_SMEM(sp); FP_SMEM(qp);
    uint32_t clo = 0, chi = 0;
    #pragma unroll 1
    for (int k = 0; k < 4; k++) {
        const uint2 sw = *reinterpret_cast<const uint2*>(sp + 8 * k), qw = *reinterpret_cast<const uint2*>(qp + 8 * k);
        const uint32_t cc = __byte_perm(code_mul4(sw.x), code_mul4(sw.y), 0x7310);
        clo = __byte_perm(clo, chi, 0x5432); chi = __byte_perm(chi, cc, 0x7632);
        const uint32_t m8 = (rmask >> (8 * k)) & 0xFFu;
        if (m8) {
            #pragma unroll
            for (int b8 = 0; b8 < 8; b8++) {
                const uint32_t w = b8 < 4 ? qw.x : qw.y;
                const int bb = b8 & 3;
                const uint32_t sh = bb == 0 ? (w << 2) : (w >> (8 * bb - 2));
                smem_dec_bit(qaddr + (sh & 0x1FCu), m8, b8);
            }
        }
    }
    /* same window arithmetic as the pre-filter items (fp_chain2_kernel phase A); a clean row's base is exact A/C/G/T iff it is not N */
    uint32_t cz = 0, cok = 0;
    if (j > 0) { cz = pack_codes4(*reinterpret_cast<const uint32_t*>(sp - 4)); cok = (~nn_prev >> 28) & 0xFu; }
    const uint32_t okm = ~nn_cur;
    const uint32_t Z0 = cz | (clo << 8), Z1 = __funnelshift_r(clo, chi, 24), Z2 = chi >> 24;
    const uint32_t O0 = cok | (okm << 4), O1 = okm >> 28;
    const uint32_t vwin = O0 & __funnelshift_r(O0, O1, 1) & __funnelshift_r(O0, O1, 2) & __funnelshift_r(O0, O1, 3) & __funnelshift_r(O0, O1, 4) & rmask;
    #pragma unroll 1
    for (int g8 = 0; g8 < 4; g8++) {
        const uint32_t v8 = (vwin >> (8 * g8)) & 0xFFu;
        if (!v8) continue;
        const uint32_t W = __funnelshift_r(g8 < 2 ? Z0 : Z1, g8 < 2 ? Z1 : Z2, (g8 & 1) * 16);
        #pragma unroll
        for (int pp = 0; pp < 8; pp++) {
            const uint32_t f4 = pp == 0 ? (W << 2) : (W >> (2 * pp - 2));
            asm volatile("red.shared.add.u32 [%0], 0xffffffff;" :: "r"((v8 & (1u << pp)) ? (kaddr | (f4 & 0xFFCu)) : kdummy) : "memory");
        }
    }
}

/* deferred post-filter statistics request (phase C): contribution of positions [lo,hi) of one tile row */
struct DeltaReq { uint32_t a, b; };        /* a = row | side<<8 | clean<<9 | (sign<0)<<10 | ctx0<<12;  b = lo | hi<<16 */

struct DeltaSinks { DeltaReq* q; int* qn; uint32_t* rm; int* nrm; int T; };
/* one region: flat lists [SIDES][T + 4], their lengths (4 words), bucket lists [SIDES][NBK][T + 4], their lengths [SIDES][NBK];
   NBK = ceil(stride / 32) */
/* removals from clean rows go to the side's removal list (fast engines); re-additions of front-shifted reads and everything on
   rows with bytes outside {A,C,G,T,N} go to the request queue (exact per-position engines) */
template <int SIDES>
__device__ __forceinline__ void push_delta(const DeltaSinks& K, bool want, bool clean, int side, int row, int ctx0, int lo, int hi, int sign) {
    if (want && hi > lo) {
        if (clean && sign < 0) {
            const int slot = atomicAdd(&K.nrm[side], 1);
            K.rm[side * (K.T + 4) + slot] = rm_pack(row, lo, hi);                  /* flat list: the histogram items of phase C */
            const int nbuckets = (c_p.stride + 31) >> 5, b = side * nbuckets + (lo >> 5);    /* bucket list: the per-cycle counters (dense_remove) */
            uint32_t* bk = K.rm + SIDES * (K.T + 4) + 4;
            int* nbk = reinterpret_cast<int*>(bk + SIDES * nbuckets * (K.T + 4));
            bk[b * (K.T + 4) + atomicAdd(&nbk[b], 1)] = rm_pack(row, lo, hi);
        } else {
            const int slot = atomicAdd(K.qn, 1);
            DeltaReq r; r.a = (uint32_t)row | ((uint32_t)side << 8) | ((clean ? 1u : 0u) << 9) | ((sign < 0 ? 1u : 0u) << 10) | ((uint32_t)ctx0 << 12); r.b = (uint32_t)lo | ((uint32_t)hi << 16);
            K.q[slot] = r;
        }
    }
}

/* ------------------------------------------------------------------------------------------------
 * The fused kernel, generation 2.  Persistent, one CTA of kChainThreads per SM, one tile at a time.  Per tile, separated by
 * CTA barriers (phase-synchronous execution: every warp of the SM runs the same region of the kernel, which keeps the
 * instruction cache warm):
 *   A  dense column pass (warps holding columns)  ||  bit planes + validation (the other warps)
 *   B  operator chain, one lane group per read / pair; post-stat requests go to a shared-memory queue
 *   C  the queue is drained by all warps (balanced), then the tile buffer is free for the next TMA load
 * ------------------------------------------------------------------------------------------------ */
static constexpr int kChainThreads = 512;         /* 16 warps: 128 registers each fill the SM's register file */
template <bool PAIRED>
__global__ void __launch_bounds__(kChainThreads, 1) fp_chain2_kernel(const fp_launch_args a) {
    extern __shared__ __align__(128) uint8_t smem[];
    constexpr int SIDES = PAIRED ? 2 : 1;
    const fp_smem_layout& sl = a.sl;
    const int S = c_p.stride, T = c_p.tile;
    const int tid = threadIdx.x, lane = lane_id(), warp = tid >> 5;
    unsigned long long* G = a.counters;
    const fp_counter_layout& L = c_p.L;

    uint64_t* mbar = reinterpret_cast<uint64_t*>(smem + sl.off_mbar);
    uint8_t* tile_seq[2]; uint8_t* tile_qual[2];
    tile_seq[0] = smem + sl.off_tile;
    tile_qual[0] = tile_seq[0] + sl.tile_array_bytes;
    tile_seq[1] = tile_qual[0] + sl.tile_array_bytes;
    tile_qual[1] = tile_seq[1] + sl.tile_array_bytes;
    uint16_t* s_len = reinterpret_cast<uint16_t*>(smem + sl.off_len);      /* [SIDES][T] */
    uint8_t* s_clean = smem + sl.off_clean;                                /* [SIDES][T] */
    unsigned int* s_kmer = reinterpret_cast<unsigned int*>(smem + sl.off_kmer);    /* [SIDES][1024] */
    unsigned int* s_qhist = reinterpret_cast<unsigned int*>(smem + sl.off_qhist);  /* [SIDES][128][FP_QH_REP] */
    BlockCounters* bc = reinterpret_cast<BlockCounters*>(smem + sl.off_bc);
    DeltaAcc D;
    D.cycles = S;
    D.cyc = reinterpret_cast<int*>(smem + sl.off_delta);
    D.kmer = reinterpret_cast<int*>(smem + sl.off_dkmer);
    D.qh = reinterpret_cast<int*>(smem + sl.off_dqh);
    uint32_t* s_rm = reinterpret_cast<uint32_t*>(smem + sl.off_rm);         /* [SIDES][T + 4] removal lists */
    int* s_nrm = reinterpret_cast<int*>(s_rm + SIDES * (T + 4));             /* [SIDES] their lengths */
    const int NBK = (S + 31) >> 5;                                           /* removal buckets per side: by lo >> 5 */
    uint32_t* s_bk = s_rm + SIDES * (T + 4) + 4;                             /* [SIDES][NBK][T + 4] */
    int* s_nbk = reinterpret_cast<int*>(s_bk + SIDES * NBK * (T + 4));       /* [SIDES][NBK] */
    DeltaSinks sinks; sinks.rm = s_rm; sinks.nrm = s_nrm; sinks.T = T;
    int16_t* s_lut = reinterpret_cast<int16_t*>(smem + sl.off_lut);
    const int PW = sl.plane_words, PSTR = sl.plane_stride;                  /* PSTR odd: conflict-free lane-group-per-row access */
    uint32_t* tile_planes = reinterpret_cast<uint32_t*>(smem + sl.off_planes);            /* [SIDES][T] rows of PSTR words */
    DeltaReq* s_queue = reinterpret_cast<DeltaReq*>(smem + sl.off_queue);   /* [SIDES * T * 2] */
    unsigned int* s_dummy = reinterpret_cast<unsigned int*>(smem + sl.off_dummy);   /* [32] write-only sink */
    int* s_qn = reinterpret_cast<int*>(smem + sl.off_next);                 /* [0] queue length, [1] pop cursor, [2] phase-A item cursor, [3] removal item cursor */
    sinks.q = s_queue; sinks.qn = &s_qn[0];
    uint32_t* s_corr = reinterpret_cast<uint32_t*>(smem + sl.off_corr);     /* [FP_CORR_CAP] base-correction work list of the tile (PE) */
    int* s_ncorr = reinterpret_cast<int*>(s_corr + FP_CORR_CAP);            /* its length */
    uint32_t* s_cm = reinterpret_cast<uint32_t*>(smem + sl.off_cm);         /* [SIDES][T][CMW] corrected positions of every row */
    const int CMW = sl.cm_words;

    if (((smem_u32(smem) + (uint32_t)sl.off_kmer) & 4095u) != 0u) __trap();   /* layout was built for another shared-window base */
    for (int i = tid; i < SIDES * T * PSTR; i += kChainThreads) tile_planes[i] = 0;
    for (int i = tid; i < SIDES * FP_KMER_BINS; i += kChainThreads) s_kmer[i] = 0;
    for (int i = tid; i < SIDES * FP_QUAL_BINS * FP_QH_REP; i += kChainThreads) s_qhist[i] = 0;
    for (int i = tid; i < SIDES * S * 20; i += kChainThreads) D.cyc[i] = 0;
    for (int i = tid; i < SIDES * FP_KMER_BINS; i += kChainThreads) D.kmer[i] = 0;
    for (int i = tid; i < SIDES * FP_QUAL_BINS; i += kChainThreads) D.qh[i] = 0;
    for (int i = tid; i < (int)(sizeof(BlockCounters) / 4); i += kChainThreads) reinterpret_cast<unsigned int*>(bc)[i] = 0;
    for (int i = tid; i < S + 2; i += kChainThreads) { s_lut[i] = c_p.lut_ovlimit[i]; s_lut[(S + 2) + i] = c_p.lut_lowq[i]; s_lut[2 * (S + 2) + i] = c_p.lut_mindiff[i]; }
    if (PAIRED)                                   /* --overlapped_out's diff limits: min(overlapDiffLimit, overlap_len * 0) = 0 */
        for (int i = tid; i < S + 2; i += kChainThreads) s_lut[3 * (S + 2) + i] = 0;
    if (tid == 0) { mbar_init(mbar, 1); s_qn[0] = 0; s_qn[1] = 0; s_qn[2] = 0; asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }

    /* column-pass ownership: thread = (side, half-word column): cycles 2*hc, 2*hc+1 */
    const int HPR = S >> 1;
    const int ncols = SIDES * HPR;                /* host guarantees ncols <= kChainThreads */
    const int nsplit = sl.col_split;              /* row groups are dealt round-robin to nsplit threads per column; host: 1 <= nsplit <= kChainThreads / ncols */
    const bool col_active = tid < ncols * nsplit;
    const int my_part = tid / ncols, my_col = col_active ? tid % ncols : 0;     /* my_part is read by column threads only */
    const int my_side = my_col / HPR, my_hc = my_col % HPR;
    const int my_w = my_hc >> 1, my_half = my_hc & 1;
    ColAcc2 acc;
    #pragma unroll
    for (int c = 0; c < 2; c++)
        #pragma unroll
        for (int b = 0; b < NB; b++)
            #pragma unroll
            for (int k = 0; k < 4; k++) acc.v[c][b][k] = 0;

    constexpr int GL = PAIRED ? 4 : 2;            /* lanes per unit */
    constexpr int UPW = 32 / GL;                  /* units per warp step */
    const int sub = lane % GL;
    const bool lead = sub == 0;
    const unsigned gmask = group_mask(GL);
    const int glead = lane & ~(GL - 1);

    /* stage the read lengths / clean flags of tile t (neither is read between the phase-B barrier and the end of the tile, so the
       NEXT tile's values are written during phase C and become visible with the barrier that ends it) */
    auto fill_lens = [&](long long t) {
        if (t >= a.n_tiles) return;
        const long long r0 = t * T;
        const int nr = (int)min((long long)T, a.b.n - r0);
        for (int i = tid; i < SIDES * T; i += kChainThreads) {
            const int sd = i / T, r = i % T;
            uint16_t ln = 0;
            if (r < nr) { ln = (sd == 0 ? a.b.len1 : a.b.len2)[r0 + r]; if (ln > S) ln = (uint16_t)S; }
            s_len[i] = ln;
            s_clean[i] = 1;
        }
    };
    fill_lens(blockIdx.x);
    __syncthreads();
    uint32_t parity = 0;
#ifdef FP_PHASE_TIMING
    /* measurement build (scripts/gpu_phase_timing.sh): cycles each warp of CTA 0 spends up to every barrier of a tile, summed over the launch */
    long long tph[12] = {0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0}, tlast = clock64();
#define FP_TP(k) do { const long long tn_ = clock64(); tph[k] += tn_ - tlast; tlast = tn_; } while (0)
#else
#define FP_TP(k) do { } while (0)
#endif

    #pragma unroll 1
    for (long long tix = blockIdx.x; tix < a.n_tiles; tix += gridDim.x) {
        const long long row0 = tix * T;
        const int rows = (int)min((long long)T, a.b.n - row0);
        /* ---------------- TMA bulk loads ---------------- */
        if (tid == 0) {
            asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
            const uint32_t bytes = (uint32_t)rows * (uint32_t)S;
            mbar_expect_tx(mbar, bytes * 2 * SIDES);
            tma_bulk_g2s(tile_seq[0], a.b.seq1 + row0 * S, bytes, mbar);
            tma_bulk_g2s(tile_qual[0], a.b.qual1 + row0 * S, bytes, mbar);
            if (PAIRED) {
                tma_bulk_g2s(tile_seq[1], a.b.seq2 + row0 * S, bytes, mbar);
                tma_bulk_g2s(tile_qual[1], a.b.qual2 + row0 * S, bytes, mbar);
            }
            s_qn[0] = 0; s_qn[1] = 0; s_qn[3] = 0;     /* request queue / removal items: next used after the phase-A barrier */
            if (PAIRED && c_p.correction) *s_ncorr = 0;
        }
        /* the read lengths of this tile were staged before the previous tile's last barrier (fill_lens), the bytes arrive through the
           mbarrier every thread waits on itself: no CTA barrier here */
        mbar_wait(mbar, parity);
        FP_TP(0);
        parity ^= 1;
        for (int i = tid; i < SIDES * (T + 4) + 4 + SIDES * NBK * (T + 4) + SIDES * NBK; i += kChainThreads) s_rm[i] = 0;      /* removal lists + lengths: filled in phase B */
        if (PAIRED && c_p.correction) for (int i = tid; i < SIDES * T * CMW; i += kChainThreads) s_cm[i] = 0;

        /* ---------------- phase A: dense pass (column warps) || bit planes + validation (other warps) ---------------- */
        if (col_active)           /* dense column pass: pre-filter stats of every row of the tile, two cycles per thread */
            dense_tile(acc, tile_seq[my_side], tile_qual[my_side], s_len + my_side * T, rows, S, my_w * 4, my_half, 4 * my_part, 4 * nsplit, G, my_side);
        FP_TP(10);
        {   /* bit planes + validation: 32-item batches claimed dynamically -- warps without columns start at once, the dense warps join */
            const int nwords = (S + 31) >> 5;
            const uint32_t qq4 = (uint32_t)(c_p.qualified_qual & 0x7F) * 0x01010101u;
            const uint32_t cq4 = (uint32_t)(min(max(c_p.cr_q, 0), 127)) * 0x01010101u;      /* plane 4: quality below cut_right's per-base threshold */
            const int total = SIDES * T * nwords;              /* pad words of the planes stay zero (cleared once at kernel start) */
            const bool want_cq = c_p.cut_right != 0;           /* plane 4 has one reader: cut_right */
            /* item order.  Word-major: the lanes of a warp hold the SAME word index of 32 different rows, so with reads of one length the
               row-end word (partial steps, predicated counts) is taken by whole warps instead of one lane in five.  The lanes then read
               shared memory one row pitch apart: not when the pitch is a multiple of 16 words (the 256-byte rows of 250 bp reads would
               all hit one bank) -- those tiles keep the row-major order (consecutive words of a row on consecutive lanes). */
            const bool word_major = ((S >> 2) & 15) != 0;
            const uint32_t it_div = word_major ? (uint32_t)(SIDES * T) : (uint32_t)nwords;
            const uint32_t it_magic = 0xFFFFFFFFu / it_div + 1u;             /* it / it_div == umulhi(it, magic) for it < 2^16 */
            #pragma unroll 1
            for (;;) {
                int base = 0;
                if (lane == 0) base = atomicAdd(&s_qn[2], 32);
                base = __shfl_sync(FULL_MASK, base, 0);
                if (base >= total) break;
                const int it = base + lane;
                if (it < total) {
                    const int qd = (int)__umulhi((uint32_t)it, it_magic), rd = it - qd * (int)it_div;
                    const int j = word_major ? qd : rd, rowi = word_major ? rd : qd;
                    const int sd = rowi >= T ? 1 : 0, rr2 = rowi - sd * T;
                    uint32_t lo = 0, hi = 0, nn = 0, lq = 0, cqw = 0;
                    if (rr2 < rows) {
                        const int n = (int)s_len[sd * T + rr2] - 32 * j;
                        if (n > 0) {
                            const uint8_t* tseq_sd = smem + sl.off_tile + sd * 2 * sl.tile_array_bytes; const uint8_t* tqual_sd = tseq_sd + sl.tile_array_bytes;
                            /* One pass over the chunk in four steps of 8 bases (two words): per-byte class flags of the even word in bit 0,
                               of the odd word in bit 4, so one multiply gathers 8 flags into the product's top byte (see plane_pair) and
                               PRMT shifts it into the plane word.  The same step packs the 2-bit base codes for the 5-mer windows and
                               counts the 8 qualities.  Rolled on purpose: straight-line code this size does not stay in the I-cache. */
                            const uint8_t* sp = tseq_sd + rr2 * S + 32 * j; const uint8_t* qp = tqual_sd + rr2 * S + 32 * j;
                            uint8_t* qhb = smem + sl.off_qhist;
                            /* quality histogram (stats.cpp:213): FP_QH_REP copies per bin (copy = lane & 3); bin address = q*16 | copy*4 | side*2048 */
                            const uint32_t qsel = ((uint32_t)(lane & (FP_QH_REP - 1)) << 2) | ((uint32_t)sd * (FP_QUAL_BINS * FP_QH_REP * 4));
                            const uint32_t qaddr = smem_u32(qhb) + qsel;          /* tables 2 KB-aligned: the bin offset (bits 4..10) ORs in */
                            uint32_t okm = 0, bad = 0, clo = 0, chi = 0;
                            #pragma unroll (kItemUnroll)
                            for (int k = 0; k < 4; k++) {
                                const uint2 sw = *reinterpret_cast<const uint2*>(sp + 8 * k), qw = *reinterpret_cast<const uint2*>(qp + 8 * k);
                                uint32_t f_lo, f_hi, f_nn, f_lq, f_ok, f_bad, f_cq;
                                plane_pair(sw.x, sw.y, qw.x, qw.y, qq4, f_lo, f_hi, f_nn, f_lq, f_ok, f_bad, cq4, f_cq, want_cq);
                                cqw = __byte_perm(cqw, f_cq, 0x7321);
                                lo = __byte_perm(lo, f_lo, 0x7321); hi = __byte_perm(hi, f_hi, 0x7321); nn = __byte_perm(nn, f_nn, 0x7321);
                                lq = __byte_perm(lq, f_lq, 0x7321); okm = __byte_perm(okm, f_ok, 0x7321); bad = __byte_perm(bad, f_bad, 0x7321);
                                const uint32_t cc = __byte_perm(code_mul4(sw.x), code_mul4(sw.y), 0x7310);   /* bytes 2,3 = codes of the two words */
                                clo = __byte_perm(clo, chi, 0x5432); chi = __byte_perm(chi, cc, 0x7632);
                                const int rem = n - 8 * k;                   /* valid bases from this step on */
                                if (!((qw.x | qw.y) & 0x80808080u)) {        /* every quality < 128 (else the exact loop below) */
                                    if (rem >= 8) {                          /* the usual step: all eight bases count, no predicates */
                                        #pragma unroll
                                        for (int b8 = 0; b8 < 8; b8++) {
                                            const uint32_t w = b8 < 4 ? qw.x : qw.y;
                                            const int bb = b8 & 3;
                                            const uint32_t sh = bb == 0 ? (w << 4) : (w >> (8 * bb - 4));
                                            smem_inc(qaddr | (sh & 0xFF0u));
                                        }
                                    } else {
                                        #pragma unroll
                                        for (int b8 = 0; b8 < 8; b8++) {
                                            const uint32_t w = b8 < 4 ? qw.x : qw.y;
                                            const int bb = b8 & 3;
                                            const uint32_t sh = bb == 0 ? (w << 4) : (w >> (8 * bb - 4));
                                            smem_inc_gt(qaddr | (sh & 0xFF0u), rem, b8);
                                        }
                                    }
                                } else {
                                    #pragma unroll 1
                                    for (int i = 0; i < min(rem, 8); i++) {
                                        const uint32_t qb = qp[8 * k + i];
                                        if (qb < FP_QUAL_BINS) atomicAdd(reinterpret_cast<unsigned int*>(qhb + ((qb << 4) | qsel)), 1u);
                                    }
                                }
                            }
                            const uint32_t vm = low_mask(n);
                            lo &= vm; hi &= vm; nn &= vm; lq &= vm; okm &= vm; cqw &= vm;
                            if (bad & vm) s_clean[sd * T + rr2] = 0;
                            /* pre-filter 5-mer counts (stats.cpp:228-266): a 5-mer counts iff its five bases are exact A/C/G/T.
                               Z = 2-bit codes of the 4 bases before this chunk and its 32 bases, 2 bits per base; the 5-mer ending
                               at chunk position p is the 10-bit field at bit 2p.  The table is indexed by that field (oldest base
                               in the LOW digit, code A0 C1 T2 G3); the flush maps it to the reference's index. */
                            uint32_t cz = 0, cok = 0;
                            if (j > 0) {
                                const uint32_t pw_ = *reinterpret_cast<const uint32_t*>(sp - 4);
                                cz = pack_codes4(pw_); cok = pack_nibble(exact_acgt(pw_));
                            }
                            const uint32_t Z0 = cz | (clo << 8), Z1 = __funnelshift_r(clo, chi, 24), Z2 = chi >> 24;
                            const uint32_t O0 = cok | (okm << 4), O1 = okm >> 28;
                            const uint32_t vwin = O0 & __funnelshift_r(O0, O1, 1) & __funnelshift_r(O0, O1, 2) & __funnelshift_r(O0, O1, 3) & __funnelshift_r(O0, O1, 4);
                            uint8_t* khb = smem + sl.off_kmer;
                            const uint32_t kaddr = smem_u32(khb) + (uint32_t)sd * (FP_KMER_BINS * 4);     /* 4 KB-aligned: the field (bits 2..11) ORs in */
                            const uint32_t kdummy = smem_u32(s_dummy) + 4u * (uint32_t)lane;                /* windows that do not count land here */
                            #pragma unroll (kItemUnroll)
                            for (int g8 = 0; g8 < 4; g8++) {               /* 8 windows per step: W = Z bits [16*g8, 16*g8 + 32) */
                                const uint32_t W = __funnelshift_r(g8 < 2 ? Z0 : Z1, g8 < 2 ? Z1 : Z2, (g8 & 1) * 16);
                                const uint32_t v8 = (vwin >> (8 * g8)) & 0xFFu;
                                /* one path per warp step: lanes with and without uncountable windows would otherwise run both in turn */
                                if (__all_sync(__activemask(), v8 == 0xFFu)) {      /* the usual step: eight countable windows, no selects */
                                    #pragma unroll
                                    for (int pp = 0; pp < 8; pp++) {       /* byte offset of the bin = field*4 | side*4096 */
                                        const uint32_t f4 = pp == 0 ? (W << 2) : (W >> (2 * pp - 2));
                                        smem_inc(kaddr | (f4 & 0xFFCu));
                                    }
                                } else if (__any_sync(__activemask(), v8 != 0u)) {
                                    #pragma unroll
                                    for (int pp = 0; pp < 8; pp++) {
                                        const uint32_t f4 = pp == 0 ? (W << 2) : (W >> (2 * pp - 2));
                                        smem_inc((v8 & (1u << pp)) ? (kaddr | (f4 & 0xFFCu)) : kdummy);
                                    }
                                }
                            }
                        }
                    }
                    uint32_t* pr = tile_planes + (sd * T + rr2) * PSTR + j;
                    pr[0] = lo; pr[PW] = hi; pr[2 * PW] = nn; pr[3 * PW] = lq; pr[4 * PW] = cqw;
                }
            }
        }
        FP_TP(1);
        __syncthreads();
        FP_TP(2);

        /* ---------------- phase B: operator chain, one lane GROUP per read / pair ---------------- */
        #pragma unroll 1
        for (int rb0 = 0; rb0 < rows; rb0 += (kChainThreads / 32) * UPW) { /* same trip count for every warp: the loop body holds CTA barriers */
            const int rbase = rb0 + warp * UPW;
            const int r = rbase + lane / GL;
            const bool active = r < rows;
            const int rr = active ? r : 0;
            const long long gi = row0 + rr;
            /* this step's reads / lengthSum of pre1 post1 pre2 post2: one shared add per warp and counter (bc->rl), the pre ones at once
               so that nothing of them stays live across the chain */
            auto warp_rl = [&](int k, uint32_t v) {
                v = __reduce_add_sync(FULL_MASK, v);
                if (lane == 0 && v) atomicAdd(&bc->rl[k], (unsigned long long)v);
            };
            uint32_t post[4] = {0, 0, 0, 0};              /* reads / lengthSum of post1, post2 */
            if (!PAIRED) {
                /* SingleEndProcessor::processSingleEnd loop body  seprocessor.cpp:204-296 */
                const int len0 = active ? s_len[rr] : 0;
                const bool clean = s_clean[rr] != 0;
                warp_rl(0, active && lead ? 1u : 0u); warp_rl(1, active && lead ? (uint32_t)len0 : 0u);
                TRead r1 = t_read(tile_seq[0] + rr * S, tile_planes + rr * PSTR, len0, clean);
                int flags = 0, apos = 0, abases = 0, pbase = 255, plen = 0, result = FP_FAIL_LENGTH;
                bool counted = false;
                /* filterByIndex (:220-224): after the pre-filter Stats and the duplicate check, the unit leaves; its whole row is
                   taken back out of the post-filter stats below (counted stays false) */
                const bool ixf = active && a.ix_flags && a.ix_flags[gi];
                if (ixf && lead) a.out1[gi] = t_index_filtered_result();
                if (active && !ixf) {
                    tc_apply(r1, t_trim_and_cut(r1.seq(), r1.qual(), len0, c_p.trim_front1, c_p.trim_tail1, sub, GL, clean ? r1.pl() + 4 * PW : nullptr));   /* :235 */
                    if (!r1.null && c_p.polyg && !t_polyg_cannot_trim(r1, PW, c_p.polyg_min)) { const int nl = r1.clean ? t_trim_polyg_planes(r1.pl(), PW, r1.front, r1.len, c_p.polyg_min) : t_trim_polyg(r1.seq() + r1.front, r1.len, c_p.polyg_min); if (nl != r1.len) { r1.len = nl; flags |= FP_F_POLYG_TRIMMED; } }
                    bool dimer = false;
                    if (!r1.null && c_p.adapter_enabled) {                                        /* :243-260 */
                        bool trimmed = false;
                        if (c_p.has_r1) {
                            const unsigned long long t = t_trim_by_sequence(r1, c_p.adapters + c_p.adapter_r1_off, c_p.adapter_r1_len, 4, 0, PW, bc, sub, GL, a.events, (unsigned int)gi, 0);
                            if (t) { r1.len = at_len(t); apos = at_pos(t); abases += at_bases(t); trimmed = true; }
                        }
                        if (c_p.n_fasta > 0) trimmed |= t_trim_by_multi(r1, PW, apos, abases, bc, sub, GL, a.events, (unsigned int)gi, 0);
                        if (trimmed) { if (lead) atomicAdd(&bc->fr[FP_FR_ADAPTER_READS], 1u); flags |= FP_F_ADAPTER_TRIMMED; }
                        if (trimmed && r1.len <= c_p.dimer_max_len) dimer = true;
                    }
                    if (!r1.null && c_p.polyx) {                                                  /* :263-266 */
                        const uint32_t px = t_polyx_cannot_trim(r1, PW, c_p.polyx_min) ? 0u : t_trim_polyx(r1.seq() + r1.front, r1.len, c_p.polyx_min);
                        if (px) {
                            r1.len = px_len(px); pbase = px_base(px); plen = px_n(px);
                            if (lead) { atomicAdd(&bc->fr[FP_FR_POLYX_READS + pbase], 1u); atomicAdd(&bc->fr[FP_FR_POLYX_BASES + pbase], (unsigned)plen); }
                            flags |= FP_F_POLYX_TRIMMED;
                        }
                    }
                    if (!r1.null && c_p.max_len1 > 0 && c_p.max_len1 < r1.len) r1.len = c_p.max_len1;   /* :268-271 */
                    result = t_pass_filter_pair(r1, PW, s_lut, sub, gmask);                       /* :273 */
                    if (dimer) { result = FP_FAIL_ADAPTER_DIMER; flags |= FP_F_ADAPTER_DIMER; }
                    const bool dupout = a.is_dup && a.is_dup[gi];                                 /* dedupOut :280 */
                    if (dupout) flags |= FP_F_DUPLICATE;
                    counted = !r1.null && result == FP_PASS_FILTER && !dupout;                    /* :281-286 */
                    if (lead) {
                        atomicAdd(&bc->fr[FP_FR_READSTATS + result], 1u);                          /* :278 */
                        if (counted) { post[0] += 1; post[1] += r1.len; }
                        a.out1[gi] = t_make_result(r1, result, result, flags, apos, abases, pbase, plen);
                    }
                }
                /* post stats as a delta against pre (warp-cooperative): drop what was trimmed / failed, re-add shifted windows */
                const bool keep_tail = counted && r1.front == 0;
                push_delta<SIDES>(sinks, active && lead, clean, 0, rr, 0, keep_tail ? r1.len : 0, len0, -1);
                push_delta<SIDES>(sinks, active && lead && counted && !keep_tail, clean, 0, rr, r1.front, r1.front, r1.front + r1.len, +1);
            } else {
                /* PairEndProcessor::processPairEnd loop body  peprocessor.cpp:383-643 */
                const int l1 = active ? s_len[rr] : 0, l2 = active ? s_len[T + rr] : 0;
                const bool clean1 = s_clean[rr] != 0, clean2 = s_clean[T + rr] != 0;
                warp_rl(0, active && lead ? 1u : 0u); warp_rl(1, active && lead ? (uint32_t)l1 : 0u);
                warp_rl(4, active && lead ? 1u : 0u); warp_rl(5, active && lead ? (uint32_t)l2 : 0u);
                TRead r1 = t_read(tile_seq[0] + rr * S, tile_planes + rr * PSTR, l1, clean1);
                TRead r2 = t_read(tile_seq[1] + rr * S, tile_planes + (T + rr) * PSTR, l2, clean2);
                int flags1 = 0, flags2 = 0, apos1 = 0, apos2 = 0, ab1 = 0, ab2 = 0, pb1 = 255, pb2 = 255, pl1n = 0, pl2n = 0;
                fp_ov_result ov; ov.overlapped = 0; ov.has_gap = 0; ov.offset = 0; ov.overlap_len = 0; ov.diff = 0;
                fp_ov_result ovA = ov;                    /* ovForAdapter */
                bool both = false, need_correct = false;
                /* filterByIndex (:404-410): the unit skips the chain but still reaches the CTA barriers of the correction round; its
                   rows are taken back out of the post-filter stats below (counted stays false) */
                const bool ixf = active && a.ix_flags && a.ix_flags[gi];
                const bool run = active && !ixf;
                if (ixf && lead) {
                    a.out1[gi] = t_index_filtered_result(); a.out2[gi] = t_index_filtered_result();
                    if (a.ov) a.ov[gi] = ov;
                    if (a.ovx) { fp_overlapped_result ox; ox.overlapped = 0; ox._pad = 0; ox.offset = 0; ox.overlap_len = 0; ox.r1_len = 0; a.ovx[gi] = ox; }
                }
                if (run) {
                    tc_apply(r1, t_trim_and_cut(r1.seq(), r1.qual(), l1, c_p.trim_front1, c_p.trim_tail1, sub, GL, clean1 ? r1.pl() + 4 * PW : nullptr));   /* :425-426 */
                    tc_apply(r2, t_trim_and_cut(r2.seq(), r2.qual(), l2, c_p.trim_front2, c_p.trim_tail2, sub, GL, clean2 ? r2.pl() + 4 * PW : nullptr));
                    both = !r1.null && !r2.null;
                    if (both && c_p.polyg) {                                                      /* :428-431 */
                        if (!t_polyg_cannot_trim(r1, PW, c_p.polyg_min)) { const int nl = r1.clean ? t_trim_polyg_planes(r1.pl(), PW, r1.front, r1.len, c_p.polyg_min) : t_trim_polyg(r1.seq() + r1.front, r1.len, c_p.polyg_min); if (nl != r1.len) { r1.len = nl; flags1 |= FP_F_POLYG_TRIMMED; } }
                        if (!t_polyg_cannot_trim(r2, PW, c_p.polyg_min)) { const int nl = r2.clean ? t_trim_polyg_planes(r2.pl(), PW, r2.front, r2.len, c_p.polyg_min) : t_trim_polyg(r2.seq() + r2.front, r2.len, c_p.polyg_min); if (nl != r2.len) { r2.len = nl; flags2 |= FP_F_POLYG_TRIMMED; } }
                    }
                    if (both && (c_p.adapter_enabled || c_p.correction || c_p.thread0)) {         /* :438-441 */
                        ov = (clean1 && clean2) ? t_analyze_planes(r1, r2, PW, s_lut, sub, GL) : t_analyze_bytes(r1, r2, s_lut);
                        if (c_p.thread0 && lead) {                                                /* statInsertSize :449-452 / :497-504, :710-723 */
                            int isize = c_p.isize_max;
                            if (ov.overlapped) {
                                if (ov.offset > 0) isize = r1.len + r2.len - ov.overlap_len + r1.front + r2.front;
                                else isize = ov.overlap_len + r1.front + r2.front;
                            }
                            if (isize > c_p.isize_max) isize = c_p.isize_max;
                            if (c_p.isize_max < FP_MAX_ISIZE_SMEM) atomicAdd(&bc->isize[isize], 1u);
                            else red_add64(&G[L.off_isize + isize], 1ull);
                        }
                    }
                    /* :445-447 gap-aware adapter trimming: analyze(..., allowGap) repeats the no-gap passes, then tries one gap */
                    if (both && c_p.allow_gap && (c_p.adapter_enabled || c_p.correction) && !ov.overlapped) ovA = t_analyze_gap(r1, r2, s_lut, sub, GL);
                    else ovA = ov;
                    need_correct = both && c_p.correction && !ovA.has_gap && ovA.overlapped && ovA.diff != 0;       /* :443,:453-456 */
                }
                /* ---- base correction (:453-456): the pairs' lanes decide, then the whole CTA works the tile's list, one lane per correction.
                        CTA barriers on purpose: a per-warp variant (warp-level syncs only) is slower -- warps running the
                        correction code at different times thrash the instruction cache, while
                        phase-synchronous warps share one hot region at a time. ---- */
                bool corr_overflow = false;
                const bool distributed = need_correct && clean1 && clean2;
                if (PAIRED && c_p.correction) {
                    if (distributed)
                        corr_overflow = t_correct_decide(r1, r2, PW, ovA, rr, sub, GL, s_corr, s_ncorr, FP_CORR_CAP, s_cm + rr * CMW, s_cm + (T + rr) * CMW);
                    /* the warps leave the overlap analysis at very different times, and behind this barrier they run the
                       correction code TOGETHER (one hot region of the instruction cache) */
                    FP_TP(3);
                    __syncthreads();
                    FP_TP(4);
                    const int ncorr = min(*s_ncorr, FP_CORR_CAP);
                    for (int i = tid; i < ncorr; i += kChainThreads)
                        t_correct_item(s_corr[i], tile_seq[0], sl.tile_array_bytes, S, T, s_len, s_cm, CMW, D, bc, a.sink, (unsigned int)(row0 + (s_corr[i] & 0x7F)));
                    __syncthreads();
                    for (int i = tid; i < ncorr; i += kChainThreads) {
                        const uint32_t en = s_corr[i];
                        const int erow = en & 0x7F, ewhich = (en >> 7) & 1;
                        t_correct_apply(en, tile_seq[0], sl.tile_array_bytes, S, T, tile_planes, PSTR, PW,
                                        (ewhich ? a.b.seq2 : a.b.seq1) + (row0 + erow) * S, (ewhich ? a.b.qual2 : a.b.qual1) + (row0 + erow) * S);
                    }
                    __syncthreads();
                    FP_TP(5);
                    if (tid == 0) *s_ncorr = 0;                    /* (a PE tile is one round of this loop: 16 warps x 8 pairs >= T) */
                }
                int res1 = FP_FAIL_LENGTH, res2 = FP_FAIL_LENGTH;
                bool counted = false;
                if (run) {
                    bool dimer = false;
                    if (need_correct) {
                        /* sequential path: pairs with bytes outside {A,C,G,T,N}, and what did not fit the work list (those positions still mismatch) */
                        corr_overflow = (__ballot_sync(gmask, corr_overflow) != 0u);
                        int nc = 0;
                        if ((!distributed || corr_overflow) && sub < 2)
                            nc = t_correct(r1, r2, r1.pl(), r2.pl(), PW, ovA, a.b.seq1 + gi * S + r1.front, a.b.qual1 + gi * S + r1.front,
                                           a.b.seq2 + gi * S + r2.front, a.b.qual2 + gi * S + r2.front, (unsigned int)gi, a.sink, bc, D, G, l1, l2, sub);
                        __syncwarp(gmask);                                                        /* corrected bytes / planes visible to the whole group */
                        int n2 = __shfl_sync(gmask, nc, glead), n1 = __shfl_sync(gmask, nc, glead + 1);   /* lane 0 rewrote read 2, lane 1 read 1 */
                        if (distributed) {                                                        /* + what the work list rewrote */
                            uint32_t any1 = 0, any2 = 0;
                            for (int k = 0; k < CMW; k++) { any1 |= s_cm[rr * CMW + k]; any2 |= s_cm[(T + rr) * CMW + k]; }
                            n1 += any1 ? 1 : 0; n2 += any2 ? 1 : 0;
                        }
                        if (n1 > 0) flags1 |= FP_F_CORRECTED;
                        if (n2 > 0) flags2 |= FP_F_CORRECTED;
                        if (lead && n1 + n2 > 0) atomicAdd(&bc->fr[FP_FR_CORRECTED_READS], (n1 > 0 && n2 > 0) ? 2u : 1u);   /* :75-80 */
                    }
                    if (both && c_p.adapter_enabled) {                                            /* :457-485 */
                        bool trimmed = false;
                        if (ovA.overlapped && ovA.offset < 0) {                                   /* trimByOverlapAnalysis adaptertrimmer.cpp:17-46 */
                            const int ol = ovA.overlap_len;
                            const int nl1 = min(r1.len, ol + r2.front), nl2 = min(r2.len, ol + r1.front);
                            const int a1 = r1.len - nl1, a2 = r2.len - nl2;
                            if (lead) {
                                atomicAdd(&bc->fr[FP_FR_ADAPTER_BASES], (unsigned)(a1 + a2));
                                push_event(a.events, (unsigned int)gi, 0, FP_EV_PAIR, 0, r1.front + nl1, a1, 0);      /* addAdapterTrimmed(adapter1, adapter2) */
                                push_event(a.events, (unsigned int)gi, 1, FP_EV_PAIR, 1, r2.front + nl2, a2, 0);
                            }
                            r1.len = nl1; r2.len = nl2;
                            ab1 += a1; ab2 += a2;
                            trimmed = true;
                        }
                        bool t1 = trimmed, t2 = trimmed;
                        if (!trimmed) {                                                           /* :461-466 */
                            if (c_p.has_r1) {
                                const unsigned long long t = t_trim_by_sequence(r1, c_p.adapters + c_p.adapter_r1_off, c_p.adapter_r1_len, 4, 0, PW, bc, sub, GL, a.events, (unsigned int)gi, 0);
                                t1 = t != 0ull;
                                if (t1) { r1.len = at_len(t); apos1 = at_pos(t); ab1 += at_bases(t); }
                            }
                            if (c_p.has_r2) {
                                const unsigned long long t = t_trim_by_sequence(r2, c_p.adapters + c_p.adapter_r2_off, c_p.adapter_r2_len, 4, 1, PW, bc, sub, GL, a.events, (unsigned int)gi, 1);
                                t2 = t != 0ull;
                                if (t2) { r2.len = at_len(t); apos2 = at_pos(t); ab2 += at_bases(t); }
                            }
                        }
                        if (c_p.n_fasta > 0) {                                                    /* :467-470 */
                            t1 |= t_trim_by_multi(r1, PW, apos1, ab1, bc, sub, GL, a.events, (unsigned int)gi, 0);
                            t2 |= t_trim_by_multi(r2, PW, apos2, ab2, bc, sub, GL, a.events, (unsigned int)gi, 1);
                        }
                        if (t1) { if (lead) atomicAdd(&bc->fr[FP_FR_ADAPTER_READS], 1u); flags1 |= FP_F_ADAPTER_TRIMMED; }   /* :472-475 */
                        if (t2) { if (lead) atomicAdd(&bc->fr[FP_FR_ADAPTER_READS], 1u); flags2 |= FP_F_ADAPTER_TRIMMED; }
                        if ((t1 || t2) && r1.len <= c_p.dimer_max_len && r2.len <= c_p.dimer_max_len) dimer = true;   /* :480-484 */
                    }
                    if (a.ovx) {                                                                  /* --overlapped_out :488-495 */
                        const int16_t* zlut = s_lut + 3 * (S + 2);                                /* analyze(..., diffPercentLimit 0) */
                        fp_ov_result o; o.overlapped = 0; o.offset = 0; o.overlap_len = 0;
                        if (both) o = (clean1 && clean2) ? t_analyze_planes(r1, r2, PW, zlut, sub, GL) : t_analyze_bytes(r1, r2, zlut);
                        if (lead) {
                            fp_overlapped_result ox; ox.overlapped = o.overlapped; ox._pad = 0; ox.offset = o.offset; ox.overlap_len = o.overlap_len;
                            ox.r1_len = both ? (uint16_t)r1.len : 0;
                            a.ovx[gi] = ox;
                        }
                    }
                    if (both && c_p.polyx) {                                                      /* :506-509 */
                        const uint32_t px1 = t_polyx_cannot_trim(r1, PW, c_p.polyx_min) ? 0u : t_trim_polyx(r1.seq() + r1.front, r1.len, c_p.polyx_min);
                        if (px1) {
                            r1.len = px_len(px1); pb1 = px_base(px1); pl1n = px_n(px1); flags1 |= FP_F_POLYX_TRIMMED;
                            if (lead) { atomicAdd(&bc->fr[FP_FR_POLYX_READS + pb1], 1u); atomicAdd(&bc->fr[FP_FR_POLYX_BASES + pb1], (unsigned)pl1n); }
                        }
                        const uint32_t px2 = t_polyx_cannot_trim(r2, PW, c_p.polyx_min) ? 0u : t_trim_polyx(r2.seq() + r2.front, r2.len, c_p.polyx_min);
                        if (px2) {
                            r2.len = px_len(px2); pb2 = px_base(px2); pl2n = px_n(px2); flags2 |= FP_F_POLYX_TRIMMED;
                            if (lead) { atomicAdd(&bc->fr[FP_FR_POLYX_READS + pb2], 1u); atomicAdd(&bc->fr[FP_FR_POLYX_BASES + pb2], (unsigned)pl2n); }
                        }
                    }
                    if (both) {                                                                   /* :511-516 */
                        if (c_p.max_len1 > 0 && c_p.max_len1 < r1.len) r1.len = c_p.max_len1;
                        if (c_p.max_len2 > 0 && c_p.max_len2 < r2.len) r2.len = c_p.max_len2;
                    }
                    const bool dupout = a.is_dup && a.is_dup[gi];                                 /* dedupOut :575 */
                    if (dupout) { flags1 |= FP_F_DUPLICATE; flags2 |= FP_F_DUPLICATE; }
                    int pv = 0;
                    bool merge_done = false;
                    if (c_p.merge && both) {                                                      /* merging mode :519-560 */
                        ov = (clean1 && clean2) ? t_analyze_planes(r1, r2, PW, s_lut, sub, GL) : t_analyze_bytes(r1, r2, s_lut);   /* :523, on the trimmed reads */
                        if (ov.overlapped) {
                            MView v; v.s1 = r1.seq() + r1.front; v.q1 = r1.qual() + r1.front; v.s2 = r2.seq() + r2.front; v.q2 = r2.qual() + r2.front;
                            v.n1 = ov.overlap_len + max(0, (int)ov.offset); v.n2 = ov.offset > 0 ? r2.len - ov.overlap_len : 0;
                            const int mres = t_pass_filter_view(v, sub, GL);                      /* :526 */
                            if (mres == FP_PASS_FILTER) {                                         /* :528-534 */
                                t_stat_view(G, 1, v, sub, GL);
                                if (lead) { atomicAdd(&bc->fr[FP_FR_MERGED_PAIRS], 1u); post[0] += 1; post[1] += v.n1 + v.n2; }
                            }
                            if (lead) atomicAdd(&bc->fr[FP_FR_READSTATS + mres], 2u);             /* :527 */
                            res1 = res2 = pv = mres;
                            flags1 |= FP_F_MERGED; flags2 |= FP_F_MERGED;
                            merge_done = true;
                        } else if (c_p.merge_unmerged) {                                          /* :537-560: read by read, both into read 1's post Stats */
                            res1 = t_pass_filter(r1, PW, s_lut); res2 = t_pass_filter(r2, PW, s_lut);
                            if (dimer) { res1 = res2 = FP_FAIL_ADAPTER_DIMER; flags1 |= FP_F_ADAPTER_DIMER; flags2 |= FP_F_ADAPTER_DIMER; }
                            if (lead) { atomicAdd(&bc->fr[FP_FR_READSTATS + res1], 1u); atomicAdd(&bc->fr[FP_FR_READSTATS + res2], 1u); }
                            if (res1 == FP_PASS_FILTER && !dupout) {
                                MView v; v.s1 = r1.seq() + r1.front; v.q1 = r1.qual() + r1.front; v.s2 = v.s1; v.q2 = v.q1; v.n1 = r1.len; v.n2 = 0;
                                t_stat_view(G, 1, v, sub, GL);
                                if (lead) { post[0] += 1; post[1] += r1.len; }
                            }
                            if (res2 == FP_PASS_FILTER && !dupout) {
                                MView v; v.s1 = r2.seq() + r2.front; v.q1 = r2.qual() + r2.front; v.s2 = v.s1; v.q2 = v.q1; v.n1 = r2.len; v.n2 = 0;
                                t_stat_view(G, 1, v, sub, GL);
                                if (lead) { post[0] += 1; post[1] += r2.len; }
                            }
                            pv = max(res1, res2);
                            merge_done = true;
                        }
                    }
                    if (!merge_done) {
                        {   /* :565-566: lanes 0, 1 filter read 1, lanes 2, 3 read 2 */
                            const int mine = t_pass_filter_pair(sub < 2 ? r1 : r2, PW, s_lut, sub & 1, gmask);
                            res1 = __shfl_sync(gmask, mine, glead); res2 = __shfl_sync(gmask, mine, glead + 2);
                        }
                        if (dimer) { res1 = res2 = FP_FAIL_ADAPTER_DIMER; flags1 |= FP_F_ADAPTER_DIMER; flags2 |= FP_F_ADAPTER_DIMER; }
                        pv = max(res1, res2);
                        /* merging mode keeps the post-filter Stats for merged (and --include_unmerged) reads only (:588-591) */
                        counted = !c_p.merge && !r1.null && res1 == FP_PASS_FILTER && !r2.null && res2 == FP_PASS_FILTER && !dupout;   /* :577-591 */
                        if (lead) atomicAdd(&bc->fr[FP_FR_READSTATS + pv], 2u);                   /* :573 */
                    }
                    if (lead) {
                        if (counted) { post[0] += 1; post[1] += r1.len; post[2] += 1; post[3] += r2.len; }
                        a.out1[gi] = t_make_result(r1, res1, pv, flags1, apos1, ab1, pb1, pl1n);
                        a.out2[gi] = t_make_result(r2, res2, pv, flags2, apos2, ab2, pb2, pl2n);
                        if (a.ov) a.ov[gi] = ov;
                    }
                }
                /* post stats as a delta against pre, per side (warp-cooperative) */
                {
                    const bool removed = false;        /* corrections were folded into the accumulators base by base (t_patch_delta) */
                    const bool keep1 = counted && r1.front == 0 && !removed;
                    push_delta<SIDES>(sinks, active && lead && !removed, clean1, 0, rr, 0, keep1 ? r1.len : 0, l1, -1);
                    push_delta<SIDES>(sinks, active && lead && counted && !keep1, clean1, 0, rr, r1.front, r1.front, r1.front + r1.len, +1);
                    const bool keep2 = counted && r2.front == 0 && !removed;
                    push_delta<SIDES>(sinks, active && lead && !removed, clean2, 1, rr, 0, keep2 ? r2.len : 0, l2, -1);
                    push_delta<SIDES>(sinks, active && lead && counted && !keep2, clean2, 1, rr, r2.front, r2.front, r2.front + r2.len, +1);
                }
            }
            warp_rl(2, post[0]); warp_rl(3, post[1]);
            if (PAIRED) { warp_rl(6, post[2]); warp_rl(7, post[3]); }
        }

        FP_TP(6);
        __syncthreads();
        FP_TP(7);

        /* ---------------- phase C: post-filter statistics of what the chain removed / shifted (all warps) ---------------- */
        {
            /* (1) per-cycle counters of the removal lists: the column threads, transposed dp4a pass like phase A's */
            if (col_active) {
                const int nr = s_nrm[my_side];
                if (nr > 0) dense_remove(s_bk + my_side * NBK * (T + 4), s_nbk + my_side * NBK, NBK, T + 4, my_part, nsplit, tile_seq[my_side], tile_qual[my_side], S, my_w * 4, my_half,
                                         D.cyc + my_side * S * 20, S);
            }
            FP_TP(11);
            /* (2) qualities and 5-mers of the removal lists: one lane per (entry, 32-base chunk), claimed 32 at a time */
            {
                const int nwords = (S + 31) >> 5;
                const int nr0 = s_nrm[0], nr1 = SIDES > 1 ? s_nrm[SIDES - 1] : 0;
                const int total = (nr0 + nr1) * nwords;
                const uint32_t nw_magic = 0xFFFFFFFFu / (uint32_t)nwords + 1u;
                const uint32_t kdummy = smem_u32(s_dummy) + 4u * (uint32_t)lane;
                #pragma unroll 1
                for (;;) {
                    if (total == 0) break;
                    int base = 0;
                    if (lane == 0) base = atomicAdd(&s_qn[3], 32);
                    base = __shfl_sync(FULL_MASK, base, 0);
                    if (base >= total) break;
                    const int it = base + lane;
                    if (it < total) {
                        const int ei = (int)__umulhi((uint32_t)it, nw_magic), j = it - ei * nwords;
                        const int sd = ei >= nr0 ? 1 : 0;
                        const uint32_t e = s_rm[sd * (T + 4) + ei - sd * nr0];
                        const int row = e & 0xFF, lo = (e >> 8) & 0xFFF, hi = e >> 20;
                        const int a0 = max(lo - 32 * j, 0), b0 = min(hi - 32 * j, 32);
                        if (b0 > a0) {
                            const uint8_t* sp = smem + sl.off_tile + sd * 2 * sl.tile_array_bytes + row * S + 32 * j;
                            const uint32_t* pnn = tile_planes + (sd * T + row) * PSTR + 2 * PW;
                            hist_remove_chunk(sp, sp + sl.tile_array_bytes, j, low_mask(b0) & ~low_mask(a0), pnn[j], j > 0 ? pnn[j - 1] : 0u,
                                              smem_u32(D.qh) + (uint32_t)sd * (FP_QUAL_BINS * 4), smem_u32(D.kmer) + (uint32_t)sd * (FP_KMER_BINS * 4), kdummy);
                        }
                    }
                }
            }
            /* (3) the request queue: re-additions of front-shifted reads, rows with bytes outside {A,C,G,T,N} (exact engines) */
            const int nreq = s_qn[0];
            #pragma unroll 1
            for (;;) {
                if (nreq == 0) break;
                int qi = 0;
                if (lane == 0) qi = atomicAdd(&s_qn[1], 1);
                qi = __shfl_sync(FULL_MASK, qi, 0);
                if (qi >= nreq) break;
                const DeltaReq rq = s_queue[qi];
                const int row = rq.a & 0xFF, side = (rq.a >> 8) & 1, sign = ((rq.a >> 10) & 1) ? -1 : +1;
                const int ctx0 = (int)(rq.a >> 12), rlo = (int)(rq.b & 0xFFFF), rhi = (int)(rq.b >> 16);
                const uint8_t* sq = smem + sl.off_tile + side * 2 * sl.tile_array_bytes + row * S; const uint8_t* ql = sq + sl.tile_array_bytes;
                if ((rq.a >> 9) & 1) dev_stat_positions_smem(D, side, sq, ql, ctx0, rlo, rhi, sign);
                else dev_stat_positions(G, side * 2 + 1, sq, ql, ctx0, rlo, rhi, sign);
            }
        }
        fill_lens(tix + gridDim.x);
        if (tid == 0) s_qn[2] = 0;                     /* item counter of phase A: idle since the phase-A barrier */
        FP_TP(8);
        __syncthreads();
        FP_TP(9);
    }

#ifdef FP_PHASE_TIMING
    if (blockIdx.x == 0 && lane == 0)
        printf("PHASE warp %2d col %d tma %lld colA %lld itemsA %lld totA %lld busyB1 %lld totB1 %lld corr %lld busyB2 %lld totB2 %lld colC %lld itemsC %lld totC %lld\n",
               warp, col_active ? 1 : 0, tph[0], tph[10], tph[1], tph[2], tph[3], tph[4], tph[5], tph[6], tph[7], tph[11], tph[8], tph[9]);
#endif
    __syncthreads();                               /* every warp is done with the shared tables */
    /* ---------------- flush block-level accumulators ---------------- */
    const int BIN_SLOT[NB] = {1, 3, 4, 6, 7};      /* base & 7 of A C T N G */
    if (col_active) {
        #pragma unroll
        for (int c = 0; c < 2; c++) {
            const int cyc = my_hc * 2 + c;
            if (cyc >= L.cycles) continue;
            #pragma unroll
            for (int b = 0; b < NB; b++) {
                const unsigned int n = acc.v[c][b][0], n20 = acc.v[c][b][1], n30 = acc.v[c][b][2], sq = acc.v[c][b][3];
                if (n == 0) continue;
                const long long qs = (long long)sq - 33ll * (long long)n;
                #pragma unroll 1
                for (int pp = 0; pp < 2; pp++) {       /* dense pass feeds pre AND post (post gets deltas on top) */
                    const int st = my_side * 2 + pp;
                    if (n30) red_add64(&G[fp_off_cycle(&L, st, 0 * 8 + BIN_SLOT[b], cyc)], (unsigned long long)n30);
                    if (n20) red_add64(&G[fp_off_cycle(&L, st, 1 * 8 + BIN_SLOT[b], cyc)], (unsigned long long)n20);
                    red_add64(&G[fp_off_cycle(&L, st, 2 * 8 + BIN_SLOT[b], cyc)], (unsigned long long)n);
                    red_add64(&G[fp_off_cycle(&L, st, 3 * 8 + BIN_SLOT[b], cyc)], (unsigned long long)qs);
                }
            }
        }
    }
    #pragma unroll 1
    for (int i = tid; i < SIDES * FP_KMER_BINS; i += kChainThreads) {
        const unsigned int v = s_kmer[i];
        if (v) { const int sd = i / FP_KMER_BINS, k = kmer_ref_index(i % FP_KMER_BINS); red_add64(&G[fp_off_kmer(&L, sd * 2, k)], (unsigned long long)v); red_add64(&G[fp_off_kmer(&L, sd * 2 + 1, k)], (unsigned long long)v); }
    }
    #pragma unroll 1
    for (int i = tid; i < SIDES * FP_QUAL_BINS; i += kChainThreads) {
        unsigned int v = 0;
        #pragma unroll
        for (int c = 0; c < FP_QH_REP; c++) v += s_qhist[i * FP_QH_REP + c];
        if (v) { const int sd = i / FP_QUAL_BINS, k = i % FP_QUAL_BINS; red_add64(&G[fp_off_qualhist(&L, sd * 2, k)], (unsigned long long)v); red_add64(&G[fp_off_qualhist(&L, sd * 2 + 1, k)], (unsigned long long)v); }
    }
    #pragma unroll 1
    for (int i = tid; i < SIDES * S * 20; i += kChainThreads) {
        const int v = D.cyc[i];
        if (v == 0) continue;
        const int sd = i / (S * 20), rem = i % (S * 20), cyc = rem / 20, bin = (rem % 20) / 4, kind = rem & 3;
        if (cyc >= L.cycles) continue;
        const int gk = kind == 0 ? 2 : kind == 1 ? 1 : kind == 2 ? 0 : 3;       /* count->content, q20, q30, qualsum */
        red_add64(&G[fp_off_cycle(&L, sd * 2 + 1, gk * 8 + BIN_SLOT[bin], cyc)], (unsigned long long)(long long)v);
    }
    #pragma unroll 1
    for (int i = tid; i < SIDES * FP_KMER_BINS; i += kChainThreads) { const int v = D.kmer[i]; if (v) red_add64(&G[fp_off_kmer(&L, (i / FP_KMER_BINS) * 2 + 1, kmer_ref_index(i % FP_KMER_BINS))], (unsigned long long)(long long)v); }
    #pragma unroll 1
    for (int i = tid; i < SIDES * FP_QUAL_BINS; i += kChainThreads) { const int v = D.qh[i]; if (v) red_add64(&G[fp_off_qualhist(&L, (i / FP_QUAL_BINS) * 2 + 1, i % FP_QUAL_BINS)], (unsigned long long)(long long)v); }
    #pragma unroll 1
    for (int i = tid; i < FP_FR_WORDS; i += kChainThreads) { const unsigned int v = bc->fr[i]; if (v) red_add64(&G[L.off_filter + i], (unsigned long long)v); }
    if (c_p.isize_max < FP_MAX_ISIZE_SMEM) {
        #pragma unroll 1
        for (int i = tid; i <= c_p.isize_max; i += kChainThreads) { const unsigned int v = bc->isize[i]; if (v) red_add64(&G[L.off_isize + i], (unsigned long long)v); }
    }
    if (tid < 2 * L.n_stats && tid < 8) {
        const unsigned long long v = bc->rl[tid];
        if (v) red_add64(&G[(tid & 1) ? fp_off_length_sum(&L, tid >> 1) : fp_off_reads(&L, tid >> 1)], v);
    }
}
