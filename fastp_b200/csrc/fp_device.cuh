/*
 * fp_device.cuh -- device-side building blocks of the sm_90a hot path (shared by fp_chain2.cuh):
 * the constant parameter block with the host-computed integer LUTs, bit-plane construction, the dp4a column-pass
 * accumulator, the exact per-position statistics engines (global and block-private), TMA / mbarrier wrappers,
 * the counter-finalisation kernel and the synthetic-input kernel.  The fused kernel itself is in fp_chain2.cuh.
 * Reference semantics are cited per function (file:line under /root/reference/src); SURVEY.md App. A lists the
 * quirks that are reproduced on purpose.
 */
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include "fastp_b200.h"

/* tell the compiler a pointer is a shared-memory address, so loads become LDS / atomics ATOMS instead of generic LD / ATOM */
#define FP_SMEM(p) __builtin_assume(__isShared(p))

#define FP_THREADS 256
#define FP_WARPS (FP_THREADS / 32)
#define FULL_MASK 0xffffffffu
#define FP_MAX_ISIZE_SMEM 1025

/* device-side parameter block (constant memory): fp_params + precomputed integer LUTs so that the
 * reference's three `double` predicates are evaluated on the host with its own expressions
 * (SURVEY.md App. A.9) and the device stays pure integer. */
struct fp_dev_params {
    int paired, thread0;
    int trim_front1, trim_tail1, trim_front2, trim_tail2, max_len1, max_len2;
    int cut_front, cut_tail, cut_right;
    int cf_w, cf_thr, ct_w, ct_thr, cr_w, cr_thr, cr_q;      /* thr = w*(33+Q); cr_q = 33+Q */
    int polyg, polyg_min, polyx, polyx_min;
    int adapter_enabled, has_r1, has_r2, n_fasta, fasta_match_req, dimer_max_len;
    int merge, merge_unmerged;                               /* --merge / --include_unmerged (PE) */
    int correction, ov_require, allow_gap, ov_diff_limit;   /* ov_diff_limit: upper bound of every lut_ovlimit entry */
    int qual_filter, qualified_qual, n_base_limit, avg_qual_req;
    int length_filter, length_required, length_limit;
    int complexity_filter;
    int isize_max;
    int stride, cycles, tile, n_stats;
    int adapter_r1_off, adapter_r1_len, adapter_r2_off, adapter_r2_len;   /* into adapters blob */
    /* global-memory tables */
    const int16_t* lut_ovlimit;     /* [stride+1]  min(diffLimit, (int)(ol * (pct/100.0)))  overlapanalysis.cpp:51 */
    const int16_t* lut_lowq;        /* [2*stride+1] floor(unqualifiedPercentLimit*rlen/100.0) filter.cpp:37 (merged reads included) */
    const int16_t* lut_mindiff;     /* [2*stride+1] smallest diff with diff/(len-1) >= threshold filter.cpp:65     */
    const uint8_t* adapters;        /* blob of adapter strings, each padded to a multiple of 4 + 8               */
    const int32_t* fasta_off;       /* [n_fasta] offsets into blob */
    const int32_t* fasta_len;       /* [n_fasta] */
    const uint32_t* adapter_planes; /* [2 + n_fasta][3][8] lo/hi/nn bit planes of each adapter (index 0 = r1, 1 = r2, 2+i = fasta i) */
    const uint8_t* adapter_clean;   /* [2 + n_fasta] 1 if the adapter holds only A,C,G,T,N */
    /* counter layout */
    fp_counter_layout L;
};

__constant__ fp_dev_params c_p;

/* ------------------------------------------------------------------ small helpers */
__device__ __forceinline__ int lane_id() { return threadIdx.x & 31; }
__device__ __forceinline__ int warp_id() { return threadIdx.x >> 5; }

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

/* bytes of x that are non-zero -> bit 7 of each byte */
__device__ __forceinline__ uint32_t nz_bytes(uint32_t x) {
    return (x | ((x & 0x7F7F7F7Fu) + 0x7F7F7F7Fu)) & 0x80808080u;
}
/* unaligned 32-bit little-endian load (two aligned loads + funnel shift); reads up to 7 bytes past p */
__device__ __forceinline__ uint32_t ld_u32_unaligned(const uint8_t* p) {
    uintptr_t a = reinterpret_cast<uintptr_t>(p);
    const uint32_t* w = reinterpret_cast<const uint32_t*>(a & ~(uintptr_t)3);
    uint32_t lo = w[0], hi = w[1];
    return __funnelshift_r(lo, hi, (unsigned)(a & 3) * 8);
}
/* fire-and-forget 64-bit add to the global counter block (two's complement for negative deltas): RED, not ATOM */
__device__ __forceinline__ void red_add64(unsigned long long* p, unsigned long long v) {
    asm volatile("red.global.add.u64 [%0], %1;" ::"l"(__cvta_generic_to_global(p)), "l"(v) : "memory");
}
__device__ __forceinline__ uint8_t dev_complement(uint8_t b) {   /* util.h:16-33 */
    switch (b) {
        case 'A': case 'a': return 'T';
        case 'T': case 't': return 'A';
        case 'C': case 'c': return 'G';
        case 'G': case 'g': return 'C';
        default: return 'N';
    }
}
__device__ __forceinline__ int warp_sum(int v) {
    #pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(FULL_MASK, v, o);
    return v;
}
__device__ __forceinline__ int warp_min(int v) {
    #pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = min(v, __shfl_xor_sync(FULL_MASK, v, o));
    return v;
}

/* first i in [0,n) with pred(i) (lanes evaluate 32 consecutive i at a time), else n. warp-uniform result. */
struct BlockCounters {
    unsigned long long rl[8];      /* reads / lengthSum of pre1 post1 pre2 post2 */
    unsigned int fr[FP_FR_WORDS];
    unsigned int isize[FP_MAX_ISIZE_SMEM];
};

/* ------------------------------------------------------------------------------------------------
 * Bit planes of a read ROW (clean rows only: every base in {A,C,G,T,N}).  Bit p = row position p.
 * code = (base>>1)&3 : A0 C1 T2 G3;  lo = code bit0, hi = code bit1, both 0 under N;  nn = N mask;
 * lq = (qual < qualified_qual).  Two bases differ iff (lo^lo') | (hi^hi') | (nn^nn').
 * Each plane holds pw = stride/32 + 2 words, zero beyond the row, so any 32-bit field is one funnel
 * shift (plane_bits).  Planes of every row of a tile are built once, word-parallel (phase 0.5); users
 * address the trimmed window as bit (front + k) and mask by the current length.
 * ------------------------------------------------------------------------------------------------ */
struct Planes { uint32_t *lo, *hi, *nn, *lq; };

__device__ __forceinline__ uint32_t plane_bits(const uint32_t* P, int bit) {
    const int w = bit >> 5;
    return __funnelshift_r(P[w], P[w + 1], bit & 31);
}
__device__ __forceinline__ uint32_t low_mask(int nbits) {     /* mask of min(max(nbits,0),32) low bits */
    return nbits >= 32 ? 0xffffffffu : (nbits <= 0 ? 0u : ((1u << nbits) - 1u));
}
/* 4 bytes holding 0/1 -> 4-bit nibble, byte k -> bit k */
__device__ __forceinline__ uint32_t pack_nibble(uint32_t v01) { return ((v01 * 0x01020408u) >> 24) & 0xFu; }

/* One plane word (32 bases = 8 seq words + 8 qual words) of one row: returns false if a valid byte is outside
 * {A,C,G,T,N} or a quality has bit 7 set.  x/q: the 8 words; n = number of valid bases in this word (1..32+).
 * Words are handled in PAIRS: per-byte flags of the even word sit in bit 0 of each byte, those of the odd word in
 * bit 4, so ONE multiply gathers the 8 flags of 8 bases into the product's top byte; PRMT assembles the 32-bit word. */
__device__ __forceinline__ uint32_t gather_top4(uint32_t m0, uint32_t m1, uint32_t m2, uint32_t m3) {
    return __byte_perm(__byte_perm(m0, m1, 0x0073), __byte_perm(m2, m3, 0x0073), 0x5410);
}
/* flags of 8 bases (even word a, odd word b; qualities qa, qb): each f_* holds the 8 flags in its TOP byte
 * (bit 24+i = base i of a, bit 28+i = base i of b).  f_bad: byte outside {A,C,G,T,N} or quality bit 7 set. */
__device__ __forceinline__ void plane_pair(uint32_t a, uint32_t b, uint32_t qa, uint32_t qb, uint32_t qq4,
                                           uint32_t& f_lo, uint32_t& f_hi, uint32_t& f_nn, uint32_t& f_lq, uint32_t& f_ok, uint32_t& f_bad, uint32_t cq4, uint32_t& f_cq, bool want_cq = true) {
    const uint32_t K = 0x01010101u, K4 = 0x10101010u, M = 0x01020408u;
    /* even word: bit j of every byte moved to bit 0 */
    const uint32_t a1 = a >> 1, a2 = a >> 2, a3 = a >> 3, a4 = a >> 4;
    const uint32_t upA = ~(a >> 5) & (a >> 6) & ~(a >> 7);                           /* bits 7..5 == 010 */
    const uint32_t okA = ((a & (~a2 | a1) & ~a3 & ~a4) | (~a & ~a1 & a2 & ~a3 & a4)) & upA & K;   /* 0x41 0x43 0x47 | 0x54 */
    const uint32_t nA = ~a & a1 & a2 & a3 & ~a4 & upA & K;                           /* 0x4E */
    /* odd word: bit j of every byte moved to bit 4 */
    const uint32_t b0 = b << 4, b1 = b << 3, b2 = b << 2, b3 = b << 1;
    const uint32_t upB = ~(b >> 1) & (b >> 2) & ~(b >> 3);
    const uint32_t okB = ((b0 & (~b2 | b1) & ~b3 & ~b) | (~b0 & ~b1 & b2 & ~b3 & b)) & upB & K4;
    const uint32_t nB = ~b0 & b1 & b2 & b3 & ~b & upB & K4;
    const uint32_t okp = okA | okB, np = nA | nB;
    /* q < qualified_qual  <=>  bit7 of (q | 0x80) - qq is clear (q, qq < 128) */
    const uint32_t ta = ~((qa | 0x80808080u) - qq4), tb = ~((qb | 0x80808080u) - qq4);
    f_lo = (((a1 & K) | (b1 & K4)) & okp) * M;
    f_hi = (((a2 & K) | (b2 & K4)) & okp) * M;
    f_nn = np * M;
    f_ok = okp * M;                                                                   /* exact: byte is one of 'A','C','G','T' */
    f_lq = (((ta >> 7) & K) | ((tb >> 3) & K4)) * M;
    f_cq = 0;
    if (want_cq) {   /* q < cut_right's per-base threshold 33+Q (filter.cpp:159): a window without such a base cannot fall below w*(33+Q) */
        const uint32_t ca = ~((qa | 0x80808080u) - cq4), cb = ~((qb | 0x80808080u) - cq4);
        f_cq = (((ca >> 7) & K) | ((cb >> 3) & K4)) * M;
    }
    f_bad = ((~(okp | np) & (K | K4)) | ((qa >> 7) & K) | ((qb >> 3) & K4)) * M;
}

/* ballot-based rebuild of one row's planes (used after base correction rewrote the row; rare) */
/* sink of the base-correction patch list (fp_patch entries, capacity, running count).  Out-of-line functions take it BY VALUE: the
   kernel's copy lives in its parameter block (fp_launch_args::sink), which has no generic address, so a reference to it makes the
   compiler copy the whole block to local memory at kernel entry and read every launch argument from there (on sm_90a that cost the
   paired kernel 512 bytes of stack and 280 bytes of register spills per thread). */
struct PatchSink { fp_patch* patches; unsigned int cap; unsigned int* count; };
/* sink of the adapter-string events (fp_adapter_event entries, capacity, running count; count == nullptr: off) */
struct EventSink { fp_adapter_event* events; unsigned int cap; unsigned int* count; };
__device__ __forceinline__ void push_event(const EventSink& sk, unsigned int unit, int which, int kind, int key, int start, int len, int adapter) {
    if (!sk.count) return;
    const unsigned int slot = atomicAdd(sk.count, 1u);
    if (slot < sk.cap) {
        fp_adapter_event e;
        e.unit = unit; e.start = (uint16_t)start; e.len = (uint16_t)len; e.key = (uint16_t)key; e.which = (uint8_t)which; e.kind = (uint8_t)kind;
        e.adapter = (uint16_t)adapter; e._pad = 0;
        sk.events[slot] = e;
    }
}

/* ------------------------------------------------------------------------------------------------
 * Column-pass statistics (Stats::statRead per-base part, stats.cpp:204-268).
 *
 * Thread = (side, word column w, row group g).  It owns cycles 4w..4w+3 of that side for its whole
 * life; acc[cyc][bin][kind] are 32-bit registers: kind 0 = count, 1 = count(q>='5'), 2 = count(q>='?'),
 * 3 = sum of raw quality chars (qualsum = kind3 - 33*kind0).  Bins: A C T N G (base&7 = 1 3 4 6 7);
 * any other byte goes through a slow global-atomic path.
 * ------------------------------------------------------------------------------------------------ */
#define FP_QH_REP 4           /* copies of the block-private quality histogram (spreads same-value shared-memory atomics) */
#define NB 5
struct ColAcc { unsigned int v[4][NB][4]; };

__device__ __forceinline__ void transpose4x4(uint32_t r0, uint32_t r1, uint32_t r2, uint32_t r3,
                                             uint32_t& c0, uint32_t& c1, uint32_t& c2, uint32_t& c3) {
    uint32_t t0 = __byte_perm(r0, r1, 0x5140);   /* r0b0 r1b0 r0b1 r1b1 */
    uint32_t t1 = __byte_perm(r2, r3, 0x5140);
    uint32_t t2 = __byte_perm(r0, r1, 0x7362);   /* r0b2 r1b2 r0b3 r1b3 */
    uint32_t t3 = __byte_perm(r2, r3, 0x7362);
    c0 = __byte_perm(t0, t1, 0x5410);
    c1 = __byte_perm(t0, t1, 0x7632);
    c2 = __byte_perm(t2, t3, 0x5410);
    c3 = __byte_perm(t2, t3, 0x7632);
}

/* keep bytes [lo, hi) of the word covering positions [4w, 4w+4) */
__device__ __forceinline__ uint32_t window_mask(int w4, int lo, int hi) {
    int a = max(lo - w4, 0), b = min(hi - w4, 4);
    if (b <= a) return 0u;
    uint32_t m = (b >= 4) ? 0xffffffffu : ((1u << (8 * b)) - 1u);
    if (a > 0) m &= ~((1u << (8 * a)) - 1u);
    return m;
}

__device__ __forceinline__ void acc_cycle(unsigned int (&a)[NB][4], uint32_t s, uint32_t q) {
    /* s: bases of 4 rows at one cycle (0 = masked out), q: their quality chars */
    const uint32_t K = 0x01010101u;
    uint32_t p0 = s & K, p1 = (s >> 1) & K, p2 = (s >> 2) & K;
    uint32_t mA = p0 & ~p1 & ~p2;          /* 001 */
    uint32_t mC = p0 & p1 & ~p2;           /* 011 */
    uint32_t mT = ~p0 & ~p1 & p2;          /* 100 */
    uint32_t mN = ~p0 & p1 & p2;           /* 110 */
    uint32_t mG = p0 & p1 & p2;            /* 111 */
    /* q >= '5' (53) and q >= '?' (63): q in [0,127] -> (q + 128 - thr) bit 7 */
    uint32_t q7 = q & 0x7F7F7F7Fu;
    uint32_t t20 = ((q7 + 0x4B4B4B4Bu) >> 7) & K;   /* 128-53 = 75 = 0x4B */
    uint32_t t30 = ((q7 + 0x41414141u) >> 7) & K;   /* 128-63 = 65 = 0x41 */
    uint32_t m[NB] = {mA, mC, mT, mN, mG};
    #pragma unroll
    for (int b = 0; b < NB; b++) {
        a[b][0] = __dp4a(m[b], K, a[b][0]);
        a[b][1] = __dp4a(m[b], t20, a[b][1]);
        a[b][2] = __dp4a(m[b], t30, a[b][2]);
        a[b][3] = __dp4a(m[b], q, a[b][3]);
    }
}

__device__ __noinline__ void slow_cycle_byte(unsigned long long* G, int stats, int cycle, uint8_t base, uint8_t q);

/* acc_cycle for 4 rows that ALL reach this cycle (no window masks): bytes the register path cannot represent
 * (base&7 in {0,2,5} or quality >= 128) are found on the transposed word and take the exact global path. */
__device__ __forceinline__ void acc_cycle_full(unsigned int (&a)[NB][4], uint32_t s, uint32_t q, unsigned long long* G, int side, int cycle) {
    const uint32_t K = 0x01010101u;
    uint32_t p0 = s & K, p1 = (s >> 1) & K, p2 = (s >> 2) & K;
    const uint32_t bad = ((~p0 & ~p2) | (p0 & ~p1 & p2) | (q >> 7)) & K;
    if (bad) {
        #pragma unroll 1
        for (int k = 0; k < 4; k++)
            if ((bad >> (8 * k)) & 1u) {
                const uint8_t bb = (uint8_t)(s >> (8 * k)), qb = (uint8_t)(q >> (8 * k));
                slow_cycle_byte(G, side * 2, cycle, bb, qb);               /* dense feeds pre AND post */
                slow_cycle_byte(G, side * 2 + 1, cycle, bb, qb);
            }
        p0 &= ~bad; p1 &= ~bad; p2 &= ~bad;                                 /* 000 matches no bin */
    }
    uint32_t mA = p0 & ~p1 & ~p2, mC = p0 & p1 & ~p2, mT = ~p0 & ~p1 & p2, mN = ~p0 & p1 & p2, mG = p0 & p1 & p2;
    uint32_t q7 = q & 0x7F7F7F7Fu;
    uint32_t t20 = ((q7 + 0x4B4B4B4Bu) >> 7) & K;
    uint32_t t30 = ((q7 + 0x41414141u) >> 7) & K;
    uint32_t m[NB] = {mA, mC, mT, mN, mG};
    #pragma unroll
    for (int b = 0; b < NB; b++) {
        a[b][0] = __dp4a(m[b], K, a[b][0]);
        a[b][1] = __dp4a(m[b], t20, a[b][1]);
        a[b][2] = __dp4a(m[b], t30, a[b][2]);
        a[b][3] = __dp4a(m[b], q, a[b][3]);
    }
}

/* slow path for one byte that is not A/C/G/T/N (or a quality >= 128): global atomics */
__device__ __noinline__ void slow_cycle_byte(unsigned long long* G, int stats, int cycle, uint8_t base, uint8_t q) {
    const fp_counter_layout& L = c_p.L;
    int b = base & 7;
    if (cycle >= L.cycles) return;
    if (q >= '?') { red_add64(&G[fp_off_cycle(&L, stats, 0 * 8 + b, cycle)], 1ull); red_add64(&G[fp_off_cycle(&L, stats, 1 * 8 + b, cycle)], 1ull); }
    else if (q >= '5') red_add64(&G[fp_off_cycle(&L, stats, 1 * 8 + b, cycle)], 1ull);
    red_add64(&G[fp_off_cycle(&L, stats, 2 * 8 + b, cycle)], 1ull);
    red_add64(&G[fp_off_cycle(&L, stats, 3 * 8 + b, cycle)], (unsigned long long)(long long)((int)q - 33));
}

/* 2-bit value of a base for the 5-mer code (stats.cpp:293-318): A0 T1 C2 G3, -1 otherwise */
__device__ __forceinline__ int dev_base2val(uint8_t b) {
    return b == 'A' ? 0 : b == 'T' ? 1 : b == 'C' ? 2 : b == 'G' ? 3 : -1;
}

/* ------------------------------------------------------------------------------------------------
 * Exact per-position statistics engine (warp per row, global atomics).  Adds `sign` times the
 * contribution Stats::statRead (stats.cpp:204-268) makes for positions i in [lo,hi) of a read whose
 * first counted base is at row index ctx0 (cycle = i - ctx0; the 5-mer ending at i counts iff
 * i-4 >= ctx0 and all five bases are in ACGT).  Used for
 *   - rows holding bytes outside {A,C,G,T,N} (excluded from the dense column pass),
 *   - the post-filter Stats as a DELTA against the pre-filter Stats: post = pre - (bases removed by
 *     trimming / failed reads) + (front-shifted or corrected reads re-added).
 * ------------------------------------------------------------------------------------------------ */
__device__ __noinline__ void dev_stat_positions(unsigned long long* G, int stats, const uint8_t* seq, const uint8_t* qual,
                                               int ctx0, int lo, int hi, int sign) {
    const fp_counter_layout& L = c_p.L;
    const unsigned long long one = (unsigned long long)(long long)sign;
    for (int i = lo + lane_id(); i < hi; i += 32) {
        const uint8_t base = seq[i], q = qual[i];
        const int b = base & 7;
        const int cyc = i - ctx0;
        if (q < FP_QUAL_BINS) red_add64(&G[fp_off_qualhist(&L, stats, q)], one);
        if (cyc < L.cycles) {
            const unsigned long long qv = (unsigned long long)((long long)sign * ((int)q - 33));
            if (q >= '?') { red_add64(&G[fp_off_cycle(&L, stats, 0 * 8 + b, cyc)], one); red_add64(&G[fp_off_cycle(&L, stats, 1 * 8 + b, cyc)], one); }
            else if (q >= '5') red_add64(&G[fp_off_cycle(&L, stats, 1 * 8 + b, cyc)], one);
            red_add64(&G[fp_off_cycle(&L, stats, 2 * 8 + b, cyc)], one);
            red_add64(&G[fp_off_cycle(&L, stats, 3 * 8 + b, cyc)], qv);
        }
        if (i - 4 >= ctx0) {
            int code = 0; bool ok = true;
            #pragma unroll
            for (int k = 0; k < 5; k++) { int v = dev_base2val(seq[i - 4 + k]); ok = ok && (v >= 0); code = (code << 2) | (v & 3); }
            if (ok) red_add64(&G[fp_off_kmer(&L, stats, code)], one);
        }
    }
}

/* 2-bit codes ((base>>1)&3: A0 C1 T2 G3) of a word's 4 bases gathered into one byte: code_mul4 leaves it in byte 3 */
__device__ __forceinline__ uint32_t code_mul4(uint32_t w) { return ((w >> 1) & 0x03030303u) * 0x01041040u; }
__device__ __forceinline__ uint32_t pack_codes4(uint32_t w) { return code_mul4(w) >> 24; }

/* ------------------------------------------------------------------------------------------------
 * Block-private form of the same engine for CLEAN rows (bases in {A,C,G,T,N}): signed 32-bit shared-memory
 * accumulators instead of global atomics (the global block would serialise on its few hot addresses).
 *   D.cyc [side][cycle][bin A,C,T,N,G][kind count,q20,q30,qualsum]   D.qh [side][128]
 *   D.kmer [side][1024], indexed like the pre-filter 5-mer table (oldest base in the low digit, codes A0 C1 T2 G3)
 * Flushed once per CTA into the POST stats of that side.
 * ------------------------------------------------------------------------------------------------ */
struct DeltaAcc { int* cyc; int* kmer; int* qh; int cycles; };

__device__ __noinline__ void dev_stat_positions_smem(const DeltaAcc D, int side, const uint8_t* seq, const uint8_t* qual,
                                                    int ctx0, int lo, int hi, int sign) {
    FP_SMEM(D.cyc); FP_SMEM(D.kmer); FP_SMEM(D.qh); FP_SMEM(seq); FP_SMEM(qual);
    const int lane = lane_id();
    int* cy = D.cyc + side * D.cycles * 20;
    int* km = D.kmer + side * FP_KMER_BINS;
    int* qh = D.qh + side * FP_QUAL_BINS;
    for (int base = lo; base < hi; base += 32) {
        const int i = base + lane;
        const bool valid = i < hi;
        uint8_t b = 0, q = 0;
        if (valid) { b = seq[i]; q = qual[i]; }
        /* quality histogram: aggregate equal values inside the warp first (few distinct qualities) */
        const unsigned peers = __match_any_sync(FULL_MASK, valid ? (int)q : -1);
        if (valid && lane == __ffs(peers) - 1) atomicAdd(&qh[q], sign * __popc(peers));
        if (valid) {
            const int cyc = i - ctx0;
            if (cyc < D.cycles) {
                const int bin = (0x43F21F0Fu >> (4 * (b & 7))) & 0xF;       /* base&7: A1 C3 T4 N6 G7 -> 0..4 */
                int* c4 = cy + (cyc * 5 + bin) * 4;
                atomicAdd(&c4[0], sign);
                if (q >= '5') atomicAdd(&c4[1], sign);
                if (q >= '?') atomicAdd(&c4[2], sign);
                atomicAdd(&c4[3], sign * ((int)q - 33));
            }
            if (i - 4 >= ctx0) {
                /* 5-mer ending at i: two unaligned 32-bit loads cover bases i-4..i */
                const uint32_t w0 = ld_u32_unaligned(seq + i - 4);             /* bases i-4..i-1 */
                const uint32_t K = 0x01010101u;
                const uint32_t c0 = w0 & K, c1 = (w0 >> 1) & K, c2 = (w0 >> 2) & K;
                const uint32_t ok4 = (c0 & ~c1 & ~c2) | (c0 & c1) | (~c0 & ~c1 & c2);       /* A C G T by base&7 */
                const bool okb = (b == 'A') | (b == 'C') | (b == 'G') | (b == 'T');
                if (ok4 == K && okb) atomicAdd(&km[pack_codes4(w0) | (((uint32_t)(b >> 1) & 3u) << 8)], sign);
            }
        }
    }
}

/* post-filter delta: block-private for clean rows, exact global path otherwise */
/* ------------------------------------------------------------------------------------------------
 * Shared-memory layout of one CTA (offsets computed on the host, fp_api.cu)
 * ------------------------------------------------------------------------------------------------ */
struct fp_smem_layout {
    int off_dummy, off_mbar, off_next, off_tile, tile_array_bytes, off_len, off_clean, off_kmer, off_qhist, off_bc, off_lut, off_delta,
        off_dkmer, off_dqh, off_rm, off_planes, off_queue, plane_words, plane_stride, total,
        off_corr, off_cm, cm_words,
        col_split;                   /* threads per column of the dense column pass, 1 .. kChainThreads / (sides * stride / 2) (fp_api.cu make_smem_layout) */
};

struct fp_launch_args {
    fp_batch b;                      /* device pointers */
    fp_read_result* out1;
    fp_read_result* out2;
    fp_ov_result* ov;
    PatchSink sink;
    EventSink events;
    const uint8_t* is_dup;           /* --dedup: units flagged by the duplicate filter (nullable) */
    unsigned long long* counters;    /* global int64 block (two's complement adds) */
    long long n_tiles;
    fp_smem_layout sl;
    fp_overlapped_result* ovx;       /* --overlapped_out (PE): the exact-overlap analysis of every unit (nullable) */
    const uint8_t* ix_flags;         /* --filter_by_index1/2: units the index filter removes (nullable) */
};

__device__ __forceinline__ void mbar_init(uint64_t* bar, int count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    uint32_t ok;
    do {
        asm volatile("{\n.reg .pred p;\nmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\nselp.u32 %0, 1, 0, p;\n}\n"
                     : "=r"(ok) : "r"(smem_u32(bar)), "r"(parity) : "memory");
    } while (!ok);
}
/* TMA bulk copy global -> shared (1-D), completion signalled on the mbarrier */
__device__ __forceinline__ void tma_bulk_g2s(void* dst, const void* src, uint32_t bytes, uint64_t* bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 ::"r"(smem_u32(dst)), "l"(src), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}

/* totals per cycle (kinds 32, 33 = sum over the 8 base slots of kinds 16..23 and 24..31; stats.cpp:225-226) */
__global__ void fp_finalize_kernel(const long long* __restrict__ raw, long long* __restrict__ fin, fp_counter_layout L) {
    long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
    if (i >= L.total) return;
    long long v = raw[i];
    if (i < L.off_filter) {
        long long in_stats = i % L.stats_stride;
        int st = (int)(i / L.stats_stride);
        if (in_stats < (long long)FP_CYCLE_KINDS * L.cycles) {
            int kind = (int)(in_stats / L.cycles), cyc = (int)(in_stats % L.cycles);
            if (kind == 32 || kind == 33) {
                v = 0;
                int k0 = kind == 32 ? 16 : 24;
                for (int b = 0; b < 8; b++) v += raw[fp_off_cycle(&L, st, k0 + b, cyc)];
            }
        }
    }
    fin[i] = v;
}

/* synthetic generator: one thread per read/pair */
#include "synth.h"
__global__ void fp_synth_kernel(fp_batch b, long long first_index, unsigned long long seed, int profile, int read_len) {
    long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
    if (i >= b.n) return;
    long long o = i * b.stride;
    fp_synth_pair(seed, (uint64_t)(first_index + i), profile, read_len, b.stride, b.seq1 + o, b.qual1 + o, b.len1 + i,
                  b.seq2 ? b.seq2 + o : nullptr, b.seq2 ? b.qual2 + o : nullptr, b.seq2 ? b.len2 + i : nullptr);
}

/* ------------------------------------------------------------------------------------------------
 * Over-representation scan  (Stats::statRead, stats.cpp:270-288), its own small kernels: only 1 of every
 * `sampling` reads is scanned, so it stays out of the fused kernel.
 *   for step in {10, 20, 40, 100, min(150, evalLen-2)}:  slide i over [0, len-step); if seq[i, i+step) is a
 *   candidate: count++, dist[p]++ for p in [i, i+step) and p < evalLen, then i += step (plus the loop's i++).
 * Candidates sit in an open-addressing table keyed by a 64-bit polynomial hash of the bytes (verified byte by byte
 * on a hash hit).  One warp per sampled read: prefix hashes once, every position's substring hash in O(1), hits
 * found in parallel and then accepted in increasing i under the skip rule.
 * pre-filter stats sample by the read's global index; post-filter stats by its rank among the counted reads
 * (an exclusive scan of the verdicts, fp_overrep_rank_kernel).
 * ------------------------------------------------------------------------------------------------ */
#define FP_OVERREP_HASH_B 0x9E3779B97F4A7C15ull

struct fp_overrep_side {
    const uint8_t* blob;              /* candidate strings back to back                     */
    const int32_t* off;               /* [K] offset into blob                               */
    const int32_t* len;               /* [K]                                                */
    const unsigned long long* thash;  /* [table_size] hash of the candidate, 0 = empty slot */
    const int32_t* tidx;              /* [table_size] candidate index                       */
    int table_mask, K, eval_len;
    const uint32_t* bitmap;           /* bit (slot & bitmap_mask) set iff some slot folding there is occupied (copied to shared memory) */
    int bitmap_mask;                  /* bits - 1, bits <= FP_OVERREP_BM_BITS; -1 without candidates */
    int steps[5];                     /* 10, 20, 40, 100, min(150, eval_len - 2)            */
    unsigned long long bpow[5];       /* FP_OVERREP_HASH_B ^ steps[i]                       */
};
#define FP_OVERREP_BM_BITS 32768

struct fp_overrep_args {
    fp_batch b;
    const fp_read_result* res[2];     /* post: trimmed windows; pre: nullptr                */
    fp_overrep_side side[2];
    unsigned long long* counters;
    fp_counter_layout L;
    int post;                         /* 0: pre-filter stats (original rows), 1: post-filter stats */
    int sides, sampling;
    long long first_index;            /* pre: global index of row 0 of this batch           */
    const unsigned int* list;         /* post: batch-local indices of the sampled counted reads */
    const unsigned int* list_n;
};

static inline unsigned long long fp_overrep_pow(int step) {
    unsigned long long r = 1, b = FP_OVERREP_HASH_B;
    for (int e = step; e > 0; e >>= 1) { if (e & 1) r *= b; b *= b; }
    return r;
}

__global__ void __launch_bounds__(256) fp_overrep_kernel(const fp_overrep_args a) {
    __shared__ unsigned long long s_pref[8][FP_MAX_STRIDE + 1];
    __shared__ uint32_t s_bm[2][FP_OVERREP_BM_BITS / 32];
    /* nearly every window is no candidate: the occupancy bits of the hash table sit in shared memory, the table itself is read only
       for a window whose home slot is taken */
    for (int sd = 0; sd < a.sides; sd++)
        for (int i = threadIdx.x; i <= (a.side[sd].bitmap_mask >> 5); i += blockDim.x) s_bm[sd][i] = a.side[sd].bitmap[i];
    __syncthreads();
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const long long gw = (long long)blockIdx.x * 8 + warp;             /* one warp per (sampled read, side) */
    const long long unit = gw / a.sides;
    const int sd = (int)(gw % a.sides);
    long long row;
    if (a.post) { if (unit >= (long long)*a.list_n) return; row = a.list[unit]; }
    else {
        /* rows with (first_index + row) % sampling == 0 */
        const long long r0 = (a.sampling - (a.first_index % a.sampling)) % a.sampling;
        row = r0 + unit * a.sampling;
        if (row >= a.b.n) return;
    }
    const fp_overrep_side& S = a.side[sd];
    if (S.K == 0) return;
    const uint8_t* seq = (sd ? a.b.seq2 : a.b.seq1) + row * a.b.stride;
    int len = (sd ? a.b.len2 : a.b.len1)[row];
    if (a.post) { const fp_read_result r = a.res[sd][row]; seq += r.front; len = r.len; }
    if (len > a.b.stride) len = a.b.stride;
    unsigned long long* pref = s_pref[warp];
    {
        /* prefix hashes, 32 chunks at once: a chunk is the affine map h -> h*m + a; an inclusive warp scan of the
         * compositions gives every lane the hash in front of its chunk (same values as the serial recurrence) */
        const int c = (len + 31) >> 5;
        const int j0 = min(lane * c, len), j1 = min(j0 + c, len);
        unsigned long long m = 1, av = 0;
        for (int j = j0; j < j1; j++) { av = av * FP_OVERREP_HASH_B + (unsigned long long)(seq[j] + 1); m *= FP_OVERREP_HASH_B; }
        #pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const unsigned long long pm = __shfl_up_sync(FULL_MASK, m, o), pa = __shfl_up_sync(FULL_MASK, av, o);
            if (lane >= o) { av = pa * m + av; m = pm * m; }
        }
        unsigned long long h = __shfl_up_sync(FULL_MASK, av, 1);
        if (lane == 0) { h = 0; pref[0] = 0; }
        for (int j = j0; j < j1; j++) { h = h * FP_OVERREP_HASH_B + (unsigned long long)(seq[j] + 1); pref[j + 1] = h; }
    }
    __syncwarp();
    const int stats = sd * 2 + a.post;
    const uint32_t* bm = s_bm[sd];
    #pragma unroll 1
    for (int s5 = 0; s5 < 5; s5++) {
        const int step = S.steps[s5];
        if (step <= 0) continue;
        const unsigned long long bp = S.bpow[s5];
        const int npos = len - step;                                   /* i in [0, npos) */
        int allowed = 0;
        for (int base = 0; base < npos; base += 32) {
            const int i = base + lane;
            /* every lane: the first slot whose hash and length match (bytes not compared yet) */
            int hit = -1;
            unsigned int hslot = 0;
            unsigned long long h = 0;
            if (i < npos) {
                h = pref[i + step] - pref[i] * bp;
                if (h == 0) h = 1;
                const unsigned int home = (unsigned int)(h ^ (h >> 32)) & S.table_mask, bi = home & (unsigned int)S.bitmap_mask;
                if ((bm[bi >> 5] >> (bi & 31)) & 1u)
                    for (unsigned int slot = home;; slot = (slot + 1) & S.table_mask) {
                        const unsigned long long th = S.thash[slot];
                        if (th == 0) break;
                        if (th == h) {
                            const int k = S.tidx[slot];
                            if (S.len[k] == step) { hit = k; hslot = slot; break; }
                        }
                    }
            }
            unsigned m = __ballot_sync(FULL_MASK, hit >= 0);
            while (m) {                                                /* accept hits in increasing i under the skip rule */
                const int bit = __ffs(m) - 1;
                m &= m - 1;
                const int hi = base + bit;
                if (hi >= allowed) {
                    /* only a window that can be accepted is compared byte by byte, by the whole warp */
                    int k = __shfl_sync(FULL_MASK, hit, bit);
                    const uint8_t* c = S.blob + S.off[k];
                    bool eq = true;
                    for (int j = lane; j < step; j += 32) eq = eq && (c[j] == seq[hi + j]);
                    if (!__all_sync(FULL_MASK, eq)) {
                        /* a 64-bit hash collision: the owning lane walks on alone, comparing bytes itself */
                        if (lane == bit) {
                            hit = -1;
                            for (unsigned int slot = (hslot + 1) & S.table_mask;; slot = (slot + 1) & S.table_mask) {
                                const unsigned long long th = S.thash[slot];
                                if (th == 0) break;
                                if (th != h) continue;
                                const int k2 = S.tidx[slot];
                                if (S.len[k2] != step) continue;
                                const uint8_t* c2 = S.blob + S.off[k2];
                                bool e2 = true;
                                for (int j = 0; j < step && e2; j++) e2 = (c2[j] == seq[hi + j]);
                                if (e2) { hit = k2; break; }
                            }
                        }
                        k = __shfl_sync(FULL_MASK, hit, bit);
                        if (k < 0) continue;
                    }
                    if (lane == 0) red_add64(&a.counters[fp_off_overrep_count(&a.L, stats, k)], 1ull);
                    for (int q = hi + lane; q < hi + step && q < S.eval_len; q += 32) red_add64(&a.counters[fp_off_overrep_dist(&a.L, stats, k, q)], 1ull);
                    allowed = hi + step + 1;
                }
            }
        }
    }
}

/* rank of every counted read among the counted reads (exclusive scan of pair_verdict == PASS), in three steps;
 * emits the batch-local indices whose (base + rank) % sampling == 0 and advances *base by the batch's count. */
#define FP_RANK_ITEMS 2048
__global__ void __launch_bounds__(256) fp_overrep_blocksum_kernel(const fp_read_result* res, long long n, unsigned int* blocksum) {
    __shared__ unsigned int s[8];
    const long long b0 = (long long)blockIdx.x * FP_RANK_ITEMS;
    unsigned int c = 0;
    for (int k = threadIdx.x; k < FP_RANK_ITEMS; k += 256) { const long long i = b0 + k; if (i < n) c += (res[i].pair_verdict == FP_PASS_FILTER); }
    #pragma unroll
    for (int o = 16; o > 0; o >>= 1) c += __shfl_xor_sync(FULL_MASK, c, o);
    if ((threadIdx.x & 31) == 0) s[threadIdx.x >> 5] = c;
    __syncthreads();
    if (threadIdx.x == 0) { unsigned int t = 0; for (int w = 0; w < 8; w++) t += s[w]; blocksum[blockIdx.x] = t; }
}
__global__ void fp_overrep_scan_kernel(unsigned int* blocksum, int nblocks, unsigned long long* base, unsigned long long* base_next) {
    /* single thread: nblocks <= n / 2048 (a few tens of thousands at most); turns sums into exclusive offsets */
    if (blockIdx.x == 0 && threadIdx.x == 0) {
        unsigned long long run = 0;
        for (int i = 0; i < nblocks; i++) { const unsigned int v = blocksum[i]; blocksum[i] = (unsigned int)run; run += v; }
        *base_next = *base + run;
    }
}
__global__ void __launch_bounds__(256) fp_overrep_emit_kernel(const fp_read_result* res, long long n, const unsigned int* blockoff,
                                                              const unsigned long long* base, int sampling, unsigned int* list, unsigned int* list_n, unsigned int cap) {
    __shared__ unsigned int s_run;
    const long long b0 = (long long)blockIdx.x * FP_RANK_ITEMS;
    if (threadIdx.x == 0) s_run = blockoff[blockIdx.x];
    __syncthreads();
    const unsigned long long gbase = *base;
    for (int k0 = 0; k0 < FP_RANK_ITEMS; k0 += 256) {                  /* keep the items in order: 256 at a time */
        const long long i = b0 + k0 + threadIdx.x;
        const bool cnt = i < n && res[i].pair_verdict == FP_PASS_FILTER;
        const unsigned m = __ballot_sync(FULL_MASK, cnt);
        __shared__ unsigned int s_w[8];
        if ((threadIdx.x & 31) == 0) s_w[threadIdx.x >> 5] = __popc(m);
        __syncthreads();
        unsigned int before = s_run;
        for (int w = 0; w < (int)(threadIdx.x >> 5); w++) before += s_w[w];
        const unsigned int rank = before + __popc(m & ((1u << (threadIdx.x & 31)) - 1u));
        if (cnt && (gbase + rank) % (unsigned long long)sampling == 0) { const unsigned int slot = atomicAdd(list_n, 1u); if (slot < cap) list[slot] = (unsigned int)i; }
        __syncthreads();
        if (threadIdx.x == 0) { unsigned int t = 0; for (int w = 0; w < 8; w++) t += s_w[w]; s_run += t; }
        __syncthreads();
    }
}
