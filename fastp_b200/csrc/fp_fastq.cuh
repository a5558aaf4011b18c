/*
 * fp_fastq.cuh -- FASTQ text <-> SoA rows on the device (SURVEY.md 8(f) rank 1: the data formats either side of the hot path).
 *
 * decode  = FastqReader::getLine + FastqReader::read   src/fastqreader.cpp:240-368
 * encode  = Read::appendToString                        src/read.cpp:119-134, called for pairs/reads that pass
 *           (src/peprocessor.cpp:583-584, src/seprocessor.cpp:268)
 *
 * Semantics restated from the reference (tests/test_fastq_codec.py pins them against FastqReader itself):
 *   - a line ends at '\n' or at a '\r' that is not followed by '\n'; "\r\n" is ONE terminator and the '\r' is not content
 *     (getLine :245-266);
 *   - a record starts at the first line that is non-empty and begins with '@' (lines before it are skipped, :338-341);
 *     the next three lines are sequence, strand, quality WHATEVER they contain;
 *   - strand empty or not starting with '+' (:349), or |quality| != |sequence| (:356): the reader returns NULL, i.e. the
 *     input ENDS at that record -- the device reports the index of the first such record and the caller drops the rest;
 *   - a final line without terminator still counts (bufferFinished, :256).
 * The "which line is a record start" question is a 4-state automaton over lines (state = line position in the record);
 * it is evaluated in parallel as a scan over transition functions, so blank lines / junk between records behave
 * exactly like the sequential reader.
 *
 * Layout of the work: byte blocks of FQ_BB bytes (terminator positions), line blocks of FQ_LB lines (automaton),
 * one warp per record (scatter / gather copies).  All offsets are 32-bit: a chunk is < 4 GiB.
 */
#pragma once
#include "fp_device.cuh"

#define FQ_T 256
#define FQ_BPT 64                      /* bytes per thread in the terminator passes */
#define FQ_BB (FQ_T * FQ_BPT)          /* bytes per block */
#define FQ_LPT 8                       /* lines per thread in the automaton passes */
#define FQ_LB (FQ_T * FQ_LPT)          /* lines per block */

#define FQ_ERR_NONE 0
#define FQ_ERR_STRAND 1                /* "Expected '+'"                        fastqreader.cpp:349 */
#define FQ_ERR_LENGTH 2                /* sequence and quality differ in length fastqreader.cpp:356 */
#define FQ_ERR_STRIDE 3                /* read longer than the row stride (not a reference error: the rows are ours) */

struct fq_rec { unsigned int name_off, name_len, strand_off, strand_len; };      /* 16 B per record, offsets into the chunk */

__device__ __forceinline__ bool fq_is_term(const uint8_t* t, long long n, long long i) {
    const uint8_t c = t[i];
    return c == '\n' || (c == '\r' && (i + 1 >= n || t[i + 1] != '\n'));
}

/* ---- pass 1/2: terminator positions ---- */
__device__ __forceinline__ unsigned int fq_thread_terms(const uint8_t* text, long long n, long long b0, unsigned long long& bits) {
    /* terminator mask of this thread's FQ_BPT bytes (bit k = byte b0 + k) */
    bits = 0;
    if (b0 >= n) return 0;
    const long long e = min(b0 + (long long)FQ_BPT, n);
    if (e - b0 == FQ_BPT && ((reinterpret_cast<uintptr_t>(text + b0) & 15) == 0)) {
        const uint4* p = reinterpret_cast<const uint4*>(text + b0);
        uint8_t nextc = (e < n) ? text[e] : 0;
        #pragma unroll
        for (int v = 0; v < FQ_BPT / 16; v++) {
            const uint4 w = p[v];
            const uint32_t ws[4] = {w.x, w.y, w.z, w.w};
            #pragma unroll
            for (int k = 0; k < 4; k++) {
                #pragma unroll
                for (int b = 0; b < 4; b++) {
                    const int idx = v * 16 + k * 4 + b;
                    const uint8_t c = (uint8_t)(ws[k] >> (8 * b));
                    uint8_t nx;
                    if (b < 3) nx = (uint8_t)(ws[k] >> (8 * b + 8));
                    else if (k < 3) nx = (uint8_t)ws[k + 1];
                    else if (v + 1 < FQ_BPT / 16) nx = reinterpret_cast<const uint8_t*>(p + v + 1)[0];
                    else nx = nextc;
                    const bool last = (b0 + idx + 1 >= n);
                    if (c == '\n' || (c == '\r' && (last || nx != '\n'))) bits |= 1ull << idx;
                }
            }
        }
    } else {
        for (long long i = b0; i < e; i++) if (fq_is_term(text, n, i)) bits |= 1ull << (int)(i - b0);
    }
    return (unsigned int)__popcll(bits);
}

__device__ __forceinline__ unsigned int fq_block_excl_scan(unsigned int v, unsigned int* s_w, unsigned int& total) {
    /* exclusive prefix of v over the block's threads (FQ_T), total = block sum */
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    unsigned int inc = v;
    #pragma unroll
    for (int o = 1; o < 32; o <<= 1) { const unsigned int t = __shfl_up_sync(FULL_MASK, inc, o); if (lane >= o) inc += t; }
    if (lane == 31) s_w[w] = inc;
    __syncthreads();
    unsigned int before = 0, tot = 0;
    #pragma unroll
    for (int k = 0; k < FQ_T / 32; k++) { const unsigned int t = s_w[k]; if (k < w) before += t; tot += t; }
    __syncthreads();
    total = tot;
    return before + inc - v;
}

__global__ void __launch_bounds__(FQ_T) fq_term_count_kernel(const uint8_t* text, long long n, unsigned int* block_cnt) {
    __shared__ unsigned int s_w[FQ_T / 32];
    unsigned long long bits;
    const unsigned int c = fq_thread_terms(text, n, (long long)blockIdx.x * FQ_BB + (long long)threadIdx.x * FQ_BPT, bits);
    unsigned int tot;
    fq_block_excl_scan(c, s_w, tot);
    if (threadIdx.x == 0) block_cnt[blockIdx.x] = tot;
}
/* single thread: exclusive offsets of the byte blocks; info[0] = number of lines (incl. a final unterminated line when `final`) */
__global__ void fq_term_scan_kernel(unsigned int* block_cnt, int nblocks, const uint8_t* text, long long n, int final_chunk,
                                    unsigned int* term, unsigned int term_cap, unsigned int* info) {
    if (blockIdx.x || threadIdx.x) return;
    unsigned int run = 0;
    for (int i = 0; i < nblocks; i++) { const unsigned int v = block_cnt[i]; block_cnt[i] = run; run += v; }
    info[1] = run;                                              /* terminated lines */
    unsigned int nl = run;
    if (final_chunk && n > 0 && !fq_is_term(text, n, n - 1) && !(text[n - 1] == '\r')) {
        if (run < term_cap) term[run] = (unsigned int)n;        /* virtual terminator after the last byte */
        nl = run + 1;
    }
    info[0] = nl;
}
__global__ void __launch_bounds__(FQ_T) fq_term_fill_kernel(const uint8_t* text, long long n, const unsigned int* block_off,
                                                            unsigned int* term, unsigned int term_cap) {
    __shared__ unsigned int s_w[FQ_T / 32];
    unsigned long long bits;
    const long long b0 = (long long)blockIdx.x * FQ_BB + (long long)threadIdx.x * FQ_BPT;
    const unsigned int c = fq_thread_terms(text, n, b0, bits);
    unsigned int tot;
    unsigned int k = block_off[blockIdx.x] + fq_block_excl_scan(c, s_w, tot);
    while (bits) {
        const int b = __ffsll((long long)bits) - 1;
        bits &= bits - 1;
        if (k < term_cap) term[k] = (unsigned int)(b0 + b);
        k++;
    }
}

/* ---- line helpers ---- */
__device__ __forceinline__ void fq_line_span(const uint8_t* text, long long n, const unsigned int* term, unsigned int k,
                                             unsigned int& start, unsigned int& end) {
    start = k == 0 ? 0u : term[k - 1] + 1u;
    end = term[k];                                              /* position of the terminator (== n for the virtual one) */
    if ((long long)end < n && text[end] == '\n' && end > start && text[end - 1] == '\r') end--;     /* "\r\n": '\r' is not content */
}
__device__ __forceinline__ bool fq_namelike(const uint8_t* text, long long n, const unsigned int* term, unsigned int k) {
    unsigned int s, e;
    fq_line_span(text, n, term, k, s, e);
    return e > s && text[s] == '@';
}

/* transition function of the record automaton as 4 x 2 bits (F >> 2s) & 3 = next state from s; record counts per start state */
struct fq_elem { unsigned int F; unsigned int C[4]; };
__device__ __forceinline__ fq_elem fq_identity() { fq_elem e; e.F = 0xE4u; e.C[0] = e.C[1] = e.C[2] = e.C[3] = 0; return e; }   /* 3,2,1,0 */
__device__ __forceinline__ fq_elem fq_line_elem(bool namelike) {
    fq_elem e;
    e.F = namelike ? 0x39u : 0x38u;          /* s0->1 (or 0), s1->2, s2->3, s3->0 */
    e.C[0] = namelike ? 1u : 0u; e.C[1] = e.C[2] = e.C[3] = 0;
    return e;
}
/* a then b */
__device__ __forceinline__ fq_elem fq_compose(const fq_elem& a, const fq_elem& b) {
    fq_elem r; r.F = 0;
    #pragma unroll
    for (int s = 0; s < 4; s++) {
        const unsigned int m = (a.F >> (2 * s)) & 3u;
        r.F |= ((b.F >> (2 * m)) & 3u) << (2 * s);
        r.C[s] = a.C[s] + (m == 0 ? b.C[0] : m == 1 ? b.C[1] : m == 2 ? b.C[2] : b.C[3]);
    }
    return r;
}
__device__ __forceinline__ fq_elem fq_shfl_up(const fq_elem& e, int o) {
    fq_elem r;
    r.F = __shfl_up_sync(FULL_MASK, e.F, o);
    #pragma unroll
    for (int s = 0; s < 4; s++) r.C[s] = __shfl_up_sync(FULL_MASK, e.C[s], o);
    return r;
}

/* mode 0: block aggregates; mode 1: emit record start lines given the state / record base at the block start */
template <int MODE>
__global__ void __launch_bounds__(FQ_T) fq_fsm_kernel(const uint8_t* text, long long n, const unsigned int* term, unsigned int nlines,
                                                      fq_elem* block_agg, const unsigned int* block_state, const unsigned int* block_rec,
                                                      unsigned int* rec_line, unsigned int rec_cap) {
    __shared__ fq_elem s_w[FQ_T / 32];
    const unsigned int l0 = (unsigned int)blockIdx.x * FQ_LB + (unsigned int)threadIdx.x * FQ_LPT;
    unsigned int nl_mask = 0;
    fq_elem mine = fq_identity();
    #pragma unroll
    for (int k = 0; k < FQ_LPT; k++) {
        const unsigned int l = l0 + k;
        if (l < nlines) {
            const bool nm = fq_namelike(text, n, term, l);
            if (nm) nl_mask |= 1u << k;
            mine = fq_compose(mine, fq_line_elem(nm));
        }
    }
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    fq_elem inc = mine;
    #pragma unroll
    for (int o = 1; o < 32; o <<= 1) { const fq_elem t = fq_shfl_up(inc, o); if (lane >= o) inc = fq_compose(t, inc); }
    if (lane == 31) s_w[w] = inc;
    __syncthreads();
    if (MODE == 0) {
        if (threadIdx.x == 0) {
            fq_elem a = s_w[0];
            for (int k = 1; k < FQ_T / 32; k++) a = fq_compose(a, s_w[k]);
            block_agg[blockIdx.x] = a;
        }
        return;
    }
    /* exclusive prefix of this thread = (warps before) then (lanes before) */
    fq_elem pre = fq_identity();
    for (int k = 0; k < w; k++) pre = fq_compose(pre, s_w[k]);
    fq_elem lanes_before = fq_shfl_up(inc, 1);
    if (lane == 0) lanes_before = fq_identity();
    pre = fq_compose(pre, lanes_before);
    const unsigned int s0 = block_state[blockIdx.x];
    unsigned int st = (pre.F >> (2 * s0)) & 3u;
    unsigned int rec = block_rec[blockIdx.x] + pre.C[s0];
    #pragma unroll
    for (int k = 0; k < FQ_LPT; k++) {
        const unsigned int l = l0 + k;
        if (l < nlines) {
            const bool nm = (nl_mask >> k) & 1u;
            if (st == 0) { if (nm) { if (rec < rec_cap) rec_line[rec] = l; rec++; st = 1; } }
            else st = (st + 1) & 3u;
        }
    }
}
/* single thread: state and record count at every block start; info[2] = records started, info[3] = complete records */
__global__ void fq_fsm_scan_kernel(const fq_elem* block_agg, int nblocks, unsigned int* block_state, unsigned int* block_rec, unsigned int* info) {
    if (blockIdx.x || threadIdx.x) return;
    unsigned int st = 0, rec = 0;
    for (int b = 0; b < nblocks; b++) {
        block_state[b] = st; block_rec[b] = rec;
        const fq_elem a = block_agg[b];
        rec += a.C[st];
        st = (a.F >> (2 * st)) & 3u;
    }
    info[2] = rec;
    /* the last record is complete iff its quality line exists, i.e. the automaton is back in state 0 */
    info[3] = (st == 0) ? rec : (rec > 0 ? rec - 1 : 0);
}

/* ---- scatter: one warp per record ----
 * record r of the text goes to row `row`; first_bad / rec_end are indexed by r */
__device__ __forceinline__ void fq_scatter_record(const uint8_t* text, long long n, const unsigned int* term, const unsigned int* rec_line,
                                                  unsigned int r, unsigned int row, int stride, int phred64,
                                                  uint8_t* seq, uint8_t* qual, uint16_t* len, fq_rec* recs,
                                                  unsigned int* rec_end, unsigned int* first_bad, unsigned int* bad_code, int lane);
__global__ void __launch_bounds__(FQ_T) fq_scatter_kernel(const uint8_t* text, long long n, const unsigned int* term, const unsigned int* rec_line,
                                                          unsigned int nrec, int stride, int phred64,
                                                          uint8_t* seq, uint8_t* qual, uint16_t* len, fq_rec* recs,
                                                          unsigned int* rec_end, unsigned int* first_bad, unsigned int* bad_code) {
    const unsigned int r = blockIdx.x * (FQ_T / 32) + (threadIdx.x >> 5);
    if (r >= nrec) return;
    fq_scatter_record(text, n, term, rec_line, r, r, stride, phred64, seq, qual, len, recs, rec_end, first_bad, bad_code, threadIdx.x & 31);
}
/* interleaved text (--interleaved_in, FastqReaderPair::read src/fastqreader.cpp:452-460): record r is mate (r & 1) of pair r >> 1 */
struct fq_side_rows { uint8_t* seq[2]; uint8_t* qual[2]; uint16_t* len[2]; fq_rec* recs[2]; };
__global__ void __launch_bounds__(FQ_T) fq_scatter_il_kernel(const uint8_t* text, long long n, const unsigned int* term, const unsigned int* rec_line,
                                                             unsigned int nrec, int stride, int phred64, fq_side_rows S,
                                                             unsigned int* rec_end, unsigned int* first_bad, unsigned int* bad_code) {
    const unsigned int r = blockIdx.x * (FQ_T / 32) + (threadIdx.x >> 5);
    if (r >= nrec) return;
    const bool m2 = r & 1;                                      /* selects, not indexes: S stays in parameter space */
    fq_scatter_record(text, n, term, rec_line, r, r >> 1, stride, phred64, m2 ? S.seq[1] : S.seq[0], m2 ? S.qual[1] : S.qual[0],
                      m2 ? S.len[1] : S.len[0], m2 ? S.recs[1] : S.recs[0], rec_end, first_bad, bad_code, threadIdx.x & 31);
}
__device__ __forceinline__ void fq_scatter_record(const uint8_t* text, long long n, const unsigned int* term, const unsigned int* rec_line,
                                                  unsigned int r, unsigned int row, int stride, int phred64,
                                                  uint8_t* seq, uint8_t* qual, uint16_t* len, fq_rec* recs,
                                                  unsigned int* rec_end, unsigned int* first_bad, unsigned int* bad_code, int lane) {
    const unsigned int l = rec_line[r];
    unsigned int ns, ne, ss, se, ps, pe, qs, qe;
    fq_line_span(text, n, term, l, ns, ne);
    fq_line_span(text, n, term, l + 1, ss, se);
    fq_line_span(text, n, term, l + 2, ps, pe);
    fq_line_span(text, n, term, l + 3, qs, qe);
    int code = FQ_ERR_NONE;
    if (pe == ps || text[ps] != '+') code = FQ_ERR_STRAND;
    else if (qe - qs != se - ss) code = FQ_ERR_LENGTH;
    else if ((int)(se - ss) > stride) code = FQ_ERR_STRIDE;
    if (code != FQ_ERR_NONE) {
        if (lane == 0) { const unsigned int old = atomicMin(first_bad, r); if (r < old) atomicExch(bad_code, (unsigned int)code); }
        /* a later, smaller r may overwrite the code again: the host re-reads the code of first_bad through rec codes below */
    }
    const int L = code == FQ_ERR_NONE ? (int)(se - ss) : 0;
    uint8_t* srow = seq + (size_t)row * stride; uint8_t* qrow = qual + (size_t)row * stride;
    for (int i = lane; i < stride; i += 32) {
        uint8_t b = 0, q = 0;
        if (i < L) {
            b = text[ss + i]; q = text[qs + i];
            if (phred64) { const int v = (int)(signed char)q - 31; q = (uint8_t)(v < 33 ? 33 : v); }      /* read.cpp:35-39 */
        }
        srow[i] = b; qrow[i] = q;
    }
    if (lane == 0) {
        len[row] = (uint16_t)L;
        fq_rec rc; rc.name_off = ns; rc.name_len = ne - ns; rc.strand_off = ps; rc.strand_len = pe - ps;
        recs[row] = rc;
        /* first byte after this record's quality line (and its terminator) */
        const unsigned int t = term[l + 3];
        rec_end[r] = (long long)t < n ? t + 1u : (unsigned int)n;
        if (code != FQ_ERR_NONE) recs[row].name_len |= 0x80000000u | ((unsigned int)code << 28);     /* marks the record as bad */
    }
}

/* ---- finish: everything the host needs from a decode, written to (mapped) host memory by one thread ----
 * out[0] records kept, out[1] error code, out[2] error record (0xFFFFFFFF none), out[3] more, out[4] consumed bytes */
__global__ void fq_finish_kernel(const unsigned int* term, unsigned int nlines, unsigned int nterm, long long nbytes,
                                 const unsigned int* rec_line, unsigned int nstarted, unsigned int ncomplete, unsigned int nrec,
                                 const fq_rec* recs, const unsigned int* first_bad, unsigned int* out) {
    if (blockIdx.x || threadIdx.x) return;
    const unsigned int fb = nrec > 0 ? *first_bad : 0xFFFFFFFFu;
    unsigned int keep = nrec, err = FQ_ERR_NONE, more = 0;
    long long consumed;
    auto line_start = [&](unsigned int l) -> long long { return l == 0 ? 0ll : (long long)term[l - 1] + 1; };
    if (fb != 0xFFFFFFFFu) {                                   /* the reference reader stops here: fastqreader.cpp:349-364 */
        err = (recs[fb].name_len >> 28) & 7u; keep = fb; consumed = nbytes;
    } else if (ncomplete > nrec) {                             /* capacity reached: resume at the next record's name line */
        more = 1; consumed = line_start(rec_line[nrec]);
    } else if (nstarted > ncomplete) {                         /* the last record is not complete in this chunk: resume at its name line */
        consumed = line_start(rec_line[ncomplete]);
    } else {                                                   /* every complete line was a record line or skipped */
        consumed = nlines > nterm ? nbytes : (long long)term[nlines - 1] + 1;
    }
    out[0] = keep; out[1] = err; out[2] = fb; out[3] = more;
    out[4] = (unsigned int)(consumed & 0xFFFFFFFFll); out[5] = (unsigned int)(consumed >> 32);
}
/* fq_finish_kernel for interleaved text: out[0] counts PAIRS, out[2] is the first bad record's index in the text.  nrec (records
 * scattered) is even whenever capacity cut it.  The reference's pair stream ends at the first NULL of either mate (ReadPair::eof,
 * src/read.cpp:203-205), so a bad mate 2 also drops the good mate 1 before it, and a lone last record is dropped without a message. */
__global__ void fq_finish_il_kernel(const unsigned int* term, unsigned int nlines, unsigned int nterm, long long nbytes, int final_chunk,
                                    const unsigned int* rec_line, unsigned int nstarted, unsigned int ncomplete, unsigned int nrec,
                                    const fq_rec* recs1, const fq_rec* recs2, const unsigned int* first_bad, unsigned int* out) {
    if (blockIdx.x || threadIdx.x) return;
    const unsigned int fb = nrec > 0 ? *first_bad : 0xFFFFFFFFu;
    unsigned int keep = nrec >> 1, err = FQ_ERR_NONE, more = 0;
    long long consumed;
    auto line_start = [&](unsigned int l) -> long long { return l == 0 ? 0ll : (long long)term[l - 1] + 1; };
    if (fb != 0xFFFFFFFFu) {
        err = (((fb & 1u) ? recs2 : recs1)[fb >> 1].name_len >> 28) & 7u; keep = fb >> 1; consumed = nbytes;
    } else if (ncomplete > nrec) {                             /* capacity (in pairs) reached: resume at record 2 * capacity */
        more = 1; consumed = line_start(rec_line[nrec]);
    } else if (nrec & 1u) {                                    /* a lone mate 1: dropped at the end of the input, else read again with its mate */
        consumed = final_chunk ? nbytes : line_start(rec_line[nrec - 1]);
    } else if (nstarted > ncomplete) {
        consumed = line_start(rec_line[ncomplete]);
    } else {
        consumed = nlines > nterm ? nbytes : (long long)term[nlines - 1] + 1;
    }
    out[0] = keep; out[1] = err; out[2] = fb; out[3] = more;
    out[4] = (unsigned int)(consumed & 0xFFFFFFFFll); out[5] = (unsigned int)(consumed >> 32);
}
__global__ void fq_set_u32_kernel(unsigned int* p, unsigned int v) { if (!blockIdx.x && !threadIdx.x) *p = v; }
__global__ void fq_copy_u32_kernel(const unsigned int* src, unsigned int* dst) { if (!blockIdx.x && !threadIdx.x) *dst = *src; }

/* ---- encode ----
 * One size pass, one scan and one write pass serve the output streams, chosen at compile time:
 *   FQ_SEL_PLAIN   every unit whose pair verdict passes and that --dedup did not flag (peprocessor.cpp:575-584, seprocessor.cpp:268)
 *   FQ_SEL_MERGED  --merged_out: the merged read of a merged pair (peprocessor.cpp:528-534; the duplicate flag is not consulted),
 *                  or with --include_unmerged read 1 then read 2 of a pair that did not merge, each by its own verdict (:537-556)
 *   FQ_SEL_SIDE    --out1 / --out2 in merging mode: only units that took neither merging branch (:563-585)
 *   FQ_SEL_UNPAIRED1 / FQ_SEL_UNPAIRED2 / FQ_SEL_FAILED
 *                  --unpaired1 / --unpaired2 / --failed_out: what a unit that is not a flagged duplicate, and that took neither merging
 *                  branch, writes when exactly one read passes (peprocessor.cpp:594-620), or SE when the read fails (seprocessor.cpp:287-289);
 *                  see fq_reject_plan
 *   FQ_SEL_INTERLEAVED  --stdout for pairs (peprocessor.cpp:579-581, singleOutput): for every unit, read 1's record as FQ_SEL_PLAIN writes
 *                  it on out1, then read 2's as it writes it on out2 -- out1 and out2 interleaved record by record
 *   FQ_SEL_OVERLAPPED  --overlapped_out (peprocessor.cpp:488-495): one record per unit whose two reads trimAndCut kept and whose exact-overlap
 *                  analysis (fq_merge_args.ovx) found an overlap; see fq_overlapped_window
 * The primary arrays (text, recs, res, seq, qual) are read 1's for FQ_SEL_MERGED and the reject streams, and the written side's for
 * FQ_SEL_SIDE; fq_merge_args carries the other side (FQ_SEL_SIDE reads only its records). */
#define FQ_SCAN_ITEMS 2048
#define FQ_SEL_PLAIN 0
#define FQ_SEL_MERGED 1
#define FQ_SEL_SIDE 2
#define FQ_SEL_UNPAIRED1 3
#define FQ_SEL_UNPAIRED2 4
#define FQ_SEL_FAILED 5
#define FQ_SEL_INTERLEAVED 6
#define FQ_SEL_OVERLAPPED 7
struct fq_merge_args {
    const uint8_t* text2; const fq_rec* recs2; const fp_read_result* res2; const uint8_t* seq2; const uint8_t* qual2;
    const fp_ov_result* ov;
    const fp_overlapped_result* ovx;      /* --overlapped_out only */
    int include_unmerged;
    /* reject streams only: decoded lengths of both sides (a dropped read is written whole), which unpaired writers exist
       (bit 0: --unpaired1, bit 1: a separate --unpaired2), whether the ctx merges; res2 == NULL for single-end */
    const uint16_t* len1; const uint16_t* len2;
    int writers, merging;
};
/* which branch of peprocessor.cpp:519-622 a unit took, from its two records */
#define FQ_U_ORDINARY 0
#define FQ_U_MERGED 1
#define FQ_U_UNMERGED 2
__device__ __forceinline__ int fq_unit_class(const fp_read_result& a, const fp_read_result& b, int include_unmerged) {
    if (a.flags & FP_F_MERGED) return FQ_U_MERGED;                                               /* :525 */
    if (include_unmerged && !((a.flags | b.flags) & FP_F_DROPPED)) return FQ_U_UNMERGED;         /* :521 r1 && r2, :537 */
    return FQ_U_ORDINARY;
}
__device__ __forceinline__ bool fq_written(const fp_read_result& r, unsigned int verdict) { return verdict == FP_PASS_FILTER && !(r.flags & FP_F_DUPLICATE); }
__device__ __forceinline__ unsigned long long fq_record_size(const fq_rec& rc, const fp_read_result& r) {
    return (unsigned long long)(rc.name_len & 0x0FFFFFFFu) + rc.strand_len + 2ull * r.len + 4ull;
}
__device__ __forceinline__ unsigned int fq_digits(unsigned int v) { return v < 10u ? 1u : v < 100u ? 2u : v < 1000u ? 3u : v < 10000u ? 4u : 5u; }
/* " merged_<len1>_<len2>" (overlapanalysis.cpp:171): its length, and its byte t */
__device__ __forceinline__ unsigned int fq_suffix_len(unsigned int len1, unsigned int len2) { return 9u + fq_digits(len1) + fq_digits(len2); }
__device__ __forceinline__ uint8_t fq_suffix_byte(unsigned int t, unsigned int len1, unsigned int len2) {
    if (t < 8u) return (uint8_t)" merged_"[t];
    const unsigned int d1 = fq_digits(len1);
    unsigned int v, k;                                          /* digit k (from the right) of v */
    if (t < 8u + d1) { v = len1; k = 8u + d1 - 1u - t; }
    else if (t == 8u + d1) return '_';
    else { v = len2; k = 8u + d1 + fq_digits(len2) - t; }
    for (; k > 0; k--) v /= 10u;
    return (uint8_t)('0' + v % 10u);
}
/* fp_merged_lens for device code */
__device__ __forceinline__ void fq_merged_lens(const fp_ov_result& ov, int r2_len, int& len1, int& len2) {
    len1 = ov.overlap_len + (ov.offset > 0 ? ov.offset : 0);
    len2 = ov.offset > 0 ? r2_len - ov.overlap_len : 0;
}
__device__ __forceinline__ bool fq_strand_is_plus(const uint8_t* text, const fq_rec& rc) { return rc.strand_len == 1 && text[rc.strand_off] == '+'; }

/* ---- reject streams (--unpaired1 / --unpaired2 / --failed_out) ----
 * Tags are FAILED_TYPES (common.h:56-65) indexed by the verdict, plus FQ_TAG_PAIRED for the passing read of a pair whose mate failed.
 * A tagged record is Read::appendToStringWithTag (read.cpp:136-154): name line, ' ', tag, then the record as appendToString writes it.
 * The reference writes or1 / or2, the reads as trimAndCut left them in place: the kept window [front, front+len) of the row (corrected
 * bases included), or for a read trimAndCut dropped (never trimmed or corrected) the whole row [0, decoded length). */
#define FQ_TAG_PAIRED 32u
#define FQ_TAG_NONE 0xFFu
#define FQ_TAG_MAX 24
__constant__ char fq_tag_text[FQ_TAG_PAIRED + 1][FQ_TAG_MAX] = {
    "passed", "", "", "", "failed_polyx_filter", "", "", "", "failed_bad_overlap", "", "", "",
    "failed_too_many_n_bases", "", "", "", "failed_too_short", "failed_too_long", "", "", "failed_quality_filter", "", "", "",
    "failed_low_complexity", "", "", "", "failed_adapter_dimer", "", "", "", "paired_read_is_failing"};
__constant__ unsigned char fq_tag_len[FQ_TAG_PAIRED + 1] = {6, 0, 0, 0, 19, 0, 0, 0, 18, 0, 0, 0, 23, 0, 0, 0, 16, 15, 0, 0, 21, 0, 0, 0,
                                                             21, 0, 0, 0, 20, 0, 0, 0, 22};
/* The records one unit puts on one reject stream, in writing order, packed in a word: the count (0..2) in bits 0-1, then 9 bits per
 * record, its side (0 / 1) in the low bit and its tag (FQ_TAG_NONE = untagged) above. */
__device__ __forceinline__ unsigned int fq_plan1(unsigned int side, unsigned int tag) { return 1u | (side | tag << 1) << 2; }
__device__ __forceinline__ unsigned int fq_plan2(unsigned int s0, unsigned int t0, unsigned int s1, unsigned int t1) {
    return 2u | (s0 | t0 << 1) << 2 | (s1 | t1 << 1) << 11;
}
__device__ __forceinline__ unsigned int fq_plan_side(unsigned int P, int k) { return (P >> (2 + 9 * k)) & 1u; }
__device__ __forceinline__ unsigned int fq_plan_tag(unsigned int P, int k) { return (P >> (3 + 9 * k)) & 0xFFu; }
__device__ __forceinline__ bool fq_passes(const fp_read_result& r) { return !(r.flags & FP_F_DROPPED) && r.verdict == FP_PASS_FILTER; }
template <int SEL>
__device__ __forceinline__ unsigned int fq_reject_plan(const fp_read_result& a, const fq_merge_args& M, long long i) {
    if (a.flags & FP_F_DUPLICATE) return 0u;                                             /* dedupOut (seprocessor.cpp:280, peprocessor.cpp:575) */
    if (a.flags2 & FP_F2_INDEX_FILTERED) return 0u;                                      /* filterByIndex: the unit left before (seprocessor.cpp:220-224) */
    if (!M.res2) return SEL == FQ_SEL_FAILED && !fq_passes(a) ? fq_plan1(0, a.verdict) : 0u;        /* SE: seprocessor.cpp:281-289 */
    const fp_read_result& b = M.res2[i];
    if (M.merging && fq_unit_class(a, b, M.include_unmerged) != FQ_U_ORDINARY) return 0u; /* only the !mergeProcessed branch (:562) */
    const bool p1 = fq_passes(a), p2 = fq_passes(b);
    if (p1 == p2) return 0u;                                                             /* both written to out1/out2, or neither anywhere */
    const bool u1 = M.writers & 1, u2 = M.writers & 2;
    if (p1) {                                                                            /* :594-603 */
        if (SEL == FQ_SEL_UNPAIRED1) return u1 ? fq_plan1(0, FQ_TAG_NONE) : 0u;
        if (SEL == FQ_SEL_FAILED) return u1 ? fq_plan1(1, b.verdict) : fq_plan2(0, FQ_TAG_PAIRED, 1, b.verdict);
        return 0u;
    }
    if (SEL == FQ_SEL_UNPAIRED2) return u2 ? fq_plan1(1, FQ_TAG_NONE) : 0u;              /* :604-619 */
    if (SEL == FQ_SEL_UNPAIRED1) return u1 && !u2 ? fq_plan1(1, FQ_TAG_NONE) : 0u;
    return u1 || u2 ? fq_plan1(0, a.verdict) : fq_plan2(0, a.verdict, 1, FQ_TAG_PAIRED);
}
/* the row window a reject record writes: [from, from + n) */
__device__ __forceinline__ void fq_reject_window(const fp_read_result& r, unsigned int decoded_len, unsigned int& from, unsigned int& n) {
    if (r.flags & FP_F_DROPPED) { from = 0; n = decoded_len; } else { from = r.front; n = r.len; }
}
__device__ __forceinline__ unsigned long long fq_tagged_size(const fq_rec& rc, unsigned int tag, unsigned int n) {
    return (unsigned long long)(rc.name_len & 0x0FFFFFFFu) + (tag == FQ_TAG_NONE ? 0u : 1u + fq_tag_len[tag]) + rc.strand_len + 2ull * n + 4ull;
}
/* size of the record of side `side` of unit i with tag `tag` */
__device__ __forceinline__ unsigned long long fq_reject_record_size(const fq_rec* recs, const fp_read_result* res, const fq_merge_args& M,
                                                                    unsigned int side, unsigned int tag, long long i) {
    unsigned int from, n;
    fq_reject_window(side ? M.res2[i] : res[i], side ? M.len2[i] : M.len1[i], from, n);
    return fq_tagged_size(side ? M.recs2[i] : recs[i], tag, n);
}
template <int SEL>
__device__ __forceinline__ unsigned long long fq_reject_size(const fq_rec* recs, const fp_read_result* res, const fq_merge_args& M, long long i) {
    const unsigned int P = fq_reject_plan<SEL>(res[i], M, i);
    if (SEL != FQ_SEL_FAILED)                                   /* at most one untagged record, of a read that passes: its kept window */
        return P == 0u ? 0ull : fq_plan_side(P, 0) ? fq_record_size(M.recs2[i], M.res2[i]) : fq_record_size(recs[i], res[i]);
    unsigned long long s = 0;
    if ((P & 3u) > 0) s += fq_reject_record_size(recs, res, M, fq_plan_side(P, 0), fq_plan_tag(P, 0), i);
    if ((P & 3u) > 1) s += fq_reject_record_size(recs, res, M, fq_plan_side(P, 1), fq_plan_tag(P, 1), i);
    return s;
}
/* Read::appendToStringWithTag by one warp (untagged with FQ_TAG_NONE): returns the bytes written */
__device__ __forceinline__ unsigned long long fq_write_tagged(uint8_t* d, const uint8_t* text, const fq_rec& rc, unsigned int tag,
                                                              const uint8_t* srow, const uint8_t* qrow, unsigned int n, int lane) {
    uint8_t* const d0 = d;
    const unsigned int nl = rc.name_len & 0x0FFFFFFFu;
    for (unsigned int t = lane; t < nl; t += 32) d[t] = text[rc.name_off + t];
    d += nl;
    if (tag != FQ_TAG_NONE) {
        const unsigned int tl = fq_tag_len[tag];
        if (lane == 0) d[0] = ' ';
        for (unsigned int t = lane; t < tl; t += 32) d[1 + t] = (uint8_t)fq_tag_text[tag][t];
        d += 1 + tl;
    }
    if (lane == 0) d[0] = '\n';
    d += 1;
    for (unsigned int t = lane; t < n; t += 32) d[t] = srow[t];
    if (lane == 0) d[n] = '\n';
    d += n + 1;
    for (unsigned int t = lane; t < rc.strand_len; t += 32) d[t] = text[rc.strand_off + t];
    if (lane == 0) d[rc.strand_len] = '\n';
    d += rc.strand_len + 1;
    for (unsigned int t = lane; t < n; t += 32) d[t] = qrow[t];
    if (lane == 0) d[n] = '\n';
    return (unsigned long long)(d + n + 1 - d0);
}
/* the record of side `side` of unit i on a reject stream */
__device__ __forceinline__ unsigned long long fq_write_reject(uint8_t* d, const uint8_t* text, const fq_rec* recs, const fp_read_result* res,
                                                              const uint8_t* seq, const uint8_t* qual, const fq_merge_args& M,
                                                              unsigned int side, unsigned int tag, int stride, long long i, int lane) {
    unsigned int from, n;
    fq_reject_window(side ? M.res2[i] : res[i], side ? M.len2[i] : M.len1[i], from, n);
    const size_t row = (size_t)i * stride + from;
    return fq_write_tagged(d, side ? M.text2 : text, side ? M.recs2[i] : recs[i], tag, (side ? M.seq2 : seq) + row, (side ? M.qual2 : qual) + row, n, lane);
}

/* ---- --overlapped_out ----
 * The reference writes Read(r1 name, std::string(r1.seq.substr(max(0, offset)), overlap_len), r1 strand, the same of r1.qual): the
 * constructor takes overlap_len as a start position, so the record holds read 1 after the overlap, [max(0, offset) + overlap_len, r1_len)
 * of read 1 as the adapter trimmers left it.  That window starts at the record's front (polyX and max_len, which come later, only shorten
 * read 1 from its 3' end, hence r1_len in the analysis result), and the row holds its corrected bases.  Returns whether the unit writes;
 * its window is [from, from + n) of read 1's row (n may be 0). */
__device__ __forceinline__ bool fq_overlapped_window(const fp_read_result& a, const fp_read_result& b, const fp_overlapped_result& ov, unsigned int& from, unsigned int& n) {
    const unsigned int skip = (ov.offset > 0 ? (unsigned int)ov.offset : 0u) + (unsigned int)ov.overlap_len;
    from = a.front + skip;
    n = ov.r1_len > skip ? ov.r1_len - skip : 0u;
    return ov.overlapped && !((a.flags | b.flags) & FP_F_DROPPED);
}

/* bytes unit i puts on the selected stream */
template <int SEL>
__device__ __forceinline__ unsigned long long fq_unit_size(const uint8_t* text, const fq_rec* recs, const fp_read_result* res, const fq_merge_args& M, long long i) {
    if (SEL == FQ_SEL_OVERLAPPED) {
        unsigned int from, n;
        return fq_overlapped_window(res[i], M.res2[i], M.ovx[i], from, n) ? fq_tagged_size(recs[i], FQ_TAG_NONE, n) : 0ull;
    }
    if (SEL == FQ_SEL_INTERLEAVED) {
        const fp_read_result a = res[i], b = M.res2[i];
        return (fq_written(a, a.pair_verdict) ? fq_record_size(recs[i], a) : 0ull) + (fq_written(b, b.pair_verdict) ? fq_record_size(M.recs2[i], b) : 0ull);
    }
    if (SEL >= FQ_SEL_UNPAIRED1) return fq_reject_size<SEL>(recs, res, M, i);
    const fp_read_result r = res[i];
    if (SEL == FQ_SEL_PLAIN) return fq_written(r, r.pair_verdict) ? fq_record_size(recs[i], r) : 0ull;
    const fp_read_result r2 = M.res2[i];
    const int cls = fq_unit_class(r, r2, M.include_unmerged);
    if (SEL == FQ_SEL_SIDE) return cls == FQ_U_ORDINARY && fq_written(r, r.pair_verdict) ? fq_record_size(recs[i], r) : 0ull;
    if (cls == FQ_U_MERGED) {
        if (r.verdict != FP_PASS_FILTER) return 0ull;
        int len1, len2;
        fq_merged_lens(M.ov[i], r2.len, len1, len2);
        const fq_rec rc = recs[i];
        const unsigned int suf = fq_suffix_len((unsigned int)len1, (unsigned int)len2);
        return (unsigned long long)(rc.name_len & 0x0FFFFFFFu) + suf + rc.strand_len + (fq_strand_is_plus(text, rc) ? 0u : suf) + 2ull * (unsigned int)(len1 + len2) + 4ull;
    }
    if (cls == FQ_U_UNMERGED) return (fq_written(r, r.verdict) ? fq_record_size(recs[i], r) : 0ull) + (fq_written(r2, r2.verdict) ? fq_record_size(M.recs2[i], r2) : 0ull);
    return 0ull;
}
/* Read::appendToString (read.cpp:119-134) by one warp: name, kept window of the row, strand line, kept window of the qualities */
__device__ __forceinline__ void fq_write_record(uint8_t* d, const uint8_t* text, const fq_rec& rc, const fp_read_result& rr,
                                                const uint8_t* srow, const uint8_t* qrow, int lane) {
    const unsigned int nl = rc.name_len & 0x0FFFFFFFu;
    for (unsigned int t = lane; t < nl; t += 32) d[t] = text[rc.name_off + t];
    if (lane == 0) d[nl] = '\n';
    d += nl + 1;
    for (unsigned int t = lane; t < rr.len; t += 32) d[t] = srow[rr.front + t];
    if (lane == 0) d[rr.len] = '\n';
    d += rr.len + 1;
    for (unsigned int t = lane; t < rc.strand_len; t += 32) d[t] = text[rc.strand_off + t];
    if (lane == 0) d[rc.strand_len] = '\n';
    d += rc.strand_len + 1;
    for (unsigned int t = lane; t < rr.len; t += 32) d[t] = qrow[rr.front + t];
    if (lane == 0) d[rr.len] = '\n';
}
/* OverlapAnalysis::merge (overlapanalysis.cpp:148-179) by one warp: r1[0, len1) + reverse complement of r2[0, len2), qualities alike;
 * the suffix goes on the name line and, unless it is exactly "+", on the strand line (:173-175).  Lane t of the reversed part reads
 * s2[len2 - 1 - t]: consecutive lanes, consecutive addresses.  dev_complement is the reference's scalar map (simd.cpp:296-308). */
__device__ __forceinline__ void fq_write_merged(uint8_t* d, const uint8_t* text, const fq_rec& rc, bool plus, unsigned int len1, unsigned int len2,
                                                const uint8_t* s1, const uint8_t* q1, const uint8_t* s2, const uint8_t* q2, int lane) {
    const unsigned int nl = rc.name_len & 0x0FFFFFFFu, suf = fq_suffix_len(len1, len2);
    for (unsigned int t = lane; t < nl; t += 32) d[t] = text[rc.name_off + t];
    d += nl;
    for (unsigned int t = lane; t < suf; t += 32) d[t] = fq_suffix_byte(t, len1, len2);
    if (lane == 0) d[suf] = '\n';
    d += suf + 1;
    for (unsigned int t = lane; t < len1; t += 32) d[t] = s1[t];
    d += len1;
    for (unsigned int t = lane; t < len2; t += 32) d[t] = dev_complement(s2[len2 - 1 - t]);
    if (lane == 0) d[len2] = '\n';
    d += len2 + 1;
    for (unsigned int t = lane; t < rc.strand_len; t += 32) d[t] = text[rc.strand_off + t];
    d += rc.strand_len;
    if (!plus) { for (unsigned int t = lane; t < suf; t += 32) d[t] = fq_suffix_byte(t, len1, len2); d += suf; }
    if (lane == 0) d[0] = '\n';
    d += 1;
    for (unsigned int t = lane; t < len1; t += 32) d[t] = q1[t];
    d += len1;
    for (unsigned int t = lane; t < len2; t += 32) d[t] = q2[len2 - 1 - t];
    if (lane == 0) d[len2] = '\n';
}
template <int SEL>
__global__ void __launch_bounds__(FQ_T) fq_size_blocksum_kernel(const uint8_t* text, const fq_rec* recs, const fp_read_result* res, fq_merge_args M,
                                                                long long n, unsigned long long* blocksum) {
    __shared__ unsigned long long s[FQ_T / 32];
    const long long b0 = (long long)blockIdx.x * FQ_SCAN_ITEMS;
    unsigned long long c = 0;
    for (int k = threadIdx.x; k < FQ_SCAN_ITEMS; k += FQ_T) {
        const long long i = b0 + k;
        if (i < n) c += fq_unit_size<SEL>(text, recs, res, M, i);
    }
    #pragma unroll
    for (int o = 16; o > 0; o >>= 1) c += __shfl_xor_sync(FULL_MASK, c, o);
    if ((threadIdx.x & 31) == 0) s[threadIdx.x >> 5] = c;
    __syncthreads();
    if (threadIdx.x == 0) { unsigned long long t = 0; for (int w = 0; w < FQ_T / 32; w++) t += s[w]; blocksum[blockIdx.x] = t; }
}
__global__ void fq_size_scan_kernel(unsigned long long* blocksum, int nblocks, unsigned long long* total) {
    if (blockIdx.x || threadIdx.x) return;
    unsigned long long run = 0;
    for (int i = 0; i < nblocks; i++) { const unsigned long long v = blocksum[i]; blocksum[i] = run; run += v; }
    *total = run;
}
/* one warp per unit, FQ_SCAN_ITEMS units per block in order: the block's warps walk the units 8 at a time */
template <int SEL>
__global__ void __launch_bounds__(FQ_T) fq_encode_kernel(const uint8_t* text, const fq_rec* recs, const fp_read_result* res,
                                                         const uint8_t* seq, const uint8_t* qual, fq_merge_args M, int stride, long long n,
                                                         const unsigned long long* blockoff, uint8_t* out, unsigned long long out_cap) {
    __shared__ unsigned long long s_run;
    __shared__ unsigned long long s_sz[FQ_T];
    const long long b0 = (long long)blockIdx.x * FQ_SCAN_ITEMS;
    if (threadIdx.x == 0) s_run = blockoff[blockIdx.x];
    __syncthreads();
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    for (int k0 = 0; k0 < FQ_SCAN_ITEMS; k0 += FQ_T) {
        /* sizes of 256 consecutive units, exclusive scan inside the block */
        const long long i = b0 + k0 + threadIdx.x;
        const unsigned long long sz = i < n ? fq_unit_size<SEL>(text, recs, res, M, i) : 0ull;
        unsigned long long inc = sz;
        #pragma unroll
        for (int o = 1; o < 32; o <<= 1) { const unsigned long long t = __shfl_up_sync(FULL_MASK, inc, o); if (lane >= o) inc += t; }
        __shared__ unsigned long long s_w[FQ_T / 32];
        if (lane == 31) s_w[w] = inc;
        __syncthreads();
        unsigned long long before = s_run;
        for (int k = 0; k < w; k++) before += s_w[k];
        s_sz[threadIdx.x] = before + inc - sz;                       /* output offset of unit i */
        __syncthreads();
        /* copies: warp w takes units w, w+8, ... of this group */
        for (int j = w; j < FQ_T; j += FQ_T / 32) {
            const long long ri = b0 + k0 + j;
            if (ri >= n) break;
            const unsigned long long need = fq_unit_size<SEL>(text, recs, res, M, ri);
            const unsigned long long o = s_sz[j];
            if (need == 0 || o + need > out_cap) continue;            /* a unit that does not fit is skipped whole: caller sees total > cap */
            uint8_t* d = out + o;
            if (SEL == FQ_SEL_INTERLEAVED) {                           /* read 1 then read 2, each under its own side's rule */
                const size_t row = (size_t)ri * stride;
                const fp_read_result b = M.res2[ri];                 /* read 2's record ends the unit's `need` bytes */
                if (fq_written(b, b.pair_verdict)) {
                    const fq_rec rc2 = M.recs2[ri];
                    fq_write_record(d + (need - fq_record_size(rc2, b)), M.text2, rc2, b, M.seq2 + row, M.qual2 + row, lane);
                }
                const fp_read_result a = res[ri];
                if (fq_written(a, a.pair_verdict)) fq_write_record(d, text, recs[ri], a, seq + row, qual + row, lane);
                continue;
            }
            if (SEL == FQ_SEL_OVERLAPPED) {
                unsigned int from, n;
                fq_overlapped_window(res[ri], M.res2[ri], M.ovx[ri], from, n);
                const size_t row = (size_t)ri * stride + from;
                fq_write_tagged(d, text, recs[ri], FQ_TAG_NONE, seq + row, qual + row, n, lane);
                continue;
            }
            if (SEL >= FQ_SEL_UNPAIRED1) {                             /* reject streams: the unit's records in plan order */
                const unsigned int P = fq_reject_plan<SEL>(res[ri], M, ri);
                d += fq_write_reject(d, text, recs, res, seq, qual, M, fq_plan_side(P, 0), fq_plan_tag(P, 0), stride, ri, lane);
                if (SEL == FQ_SEL_FAILED && (P & 3u) > 1) fq_write_reject(d, text, recs, res, seq, qual, M, fq_plan_side(P, 1), fq_plan_tag(P, 1), stride, ri, lane);
                continue;
            }
            const fp_read_result rr = res[ri];
            const fq_rec rc = recs[ri];
            const uint8_t* srow = seq + (size_t)ri * stride;
            const uint8_t* qrow = qual + (size_t)ri * stride;
            if (SEL != FQ_SEL_MERGED) { fq_write_record(d, text, rc, rr, srow, qrow, lane); continue; }
            const fp_read_result r2 = M.res2[ri];
            const uint8_t* srow2 = M.seq2 + (size_t)ri * stride;
            const uint8_t* qrow2 = M.qual2 + (size_t)ri * stride;
            if (rr.flags & FP_F_MERGED) {
                int len1, len2;
                fq_merged_lens(M.ov[ri], r2.len, len1, len2);
                fq_write_merged(d, text, rc, fq_strand_is_plus(text, rc), (unsigned int)len1, (unsigned int)len2,
                                srow + rr.front, qrow + rr.front, srow2 + r2.front, qrow2 + r2.front, lane);
            } else {                                                  /* --include_unmerged: read 1 then read 2, each if it is written */
                if (fq_written(rr, rr.verdict)) { fq_write_record(d, text, rc, rr, srow, qrow, lane); d += fq_record_size(rc, rr); }
                if (fq_written(r2, r2.verdict)) fq_write_record(d, M.text2, M.recs2[ri], r2, srow2, qrow2, lane);
            }
        }
        __syncthreads();
        if (threadIdx.x == FQ_T - 1) s_run = s_sz[FQ_T - 1] + sz;
        __syncthreads();
    }
}

/* ---- index filter (--filter_by_index1 / --filter_by_index2; Read::firstIndex / lastIndex read.cpp:75-100, Filter::match filter.cpp:226-243) ----
 * A barcode list is packed by the host into 2-bit planes, plane-major and barcode-minor so that the lanes of a warp, one barcode each,
 * read consecutive words: words[(plane * W + w) * n + b] holds bases [32w, 32w + 32) of barcode b, bit t = base 32w + t, codes A0 C1 G2 T3
 * (plane 0 the low bit).  W = words per plane of the longest barcode (>= 1).  The list is read through the read-only cache: its size is
 * not limited by shared memory. */
struct fq_index_list { const uint32_t* words; const uint16_t* lens; int n, W; };
#define FQ_IX_WARPS 8
#define FQ_IX_MAXW (FP_INDEX_MAX_BARCODE / 32)

/* The index of one name by one warp: [s, e) of the name's bytes.  first = firstIndex, else lastIndex.  Walks the bytes from len-3 down
 * 32 at a time; lane t looks at byte hi - t, so the lowest lane holding a separator is the first one met. */
__device__ __forceinline__ void fq_index_span(const uint8_t* name, int len, bool first, int lane, int& s, int& e) {
    s = e = 0;
    if (len < 5) return;
    int plus = len;                                            /* lowest '+' met so far: firstIndex ends before it */
    for (int hi = len - 3; hi >= 0; hi -= 32) {
        const int p = hi - lane;
        const uint8_t c = p >= 0 ? name[p] : 0;
        const unsigned mc = __ballot_sync(FULL_MASK, c == ':' || (!first && c == '+'));
        const unsigned mp = __ballot_sync(FULL_MASK, c == '+');
        if (mc) {
            const int l = __ffs(mc) - 1;
            const unsigned above = mp & ((1u << l) - 1u);       /* '+' bytes met before this separator */
            if (first && above) plus = hi - (31 - __clz(above));
            s = hi - l + 1;
            e = first ? plus : len;
            return;
        }
        if (mp) plus = hi - (31 - __clz(mp));
    }
}

/* Whether any barcode of the list matches the index [s, e) of `name`; s_ix: this warp's 3 * FQ_IX_MAXW words of shared memory */
__device__ __forceinline__ bool fq_index_match(const uint8_t* name, int s, int e, const fq_index_list& L, int threshold, uint32_t* s_ix, int lane) {
    if (L.n == 0 || threshold < 0) return false;
    const int ilen = e - s;
    /* the index in the barcodes' planes, one word per step: lane t codes byte 32w + t, a ballot gathers the word; a byte outside
       A/C/G/T clears its bit of the valid plane and so always counts as a mismatch */
    for (int w = 0; w < L.W; w++) {
        const int p = 32 * w + lane;
        const uint8_t c = p < ilen ? name[s + p] : 0;
        const unsigned code = c == 'C' ? 1u : c == 'G' ? 2u : c == 'T' ? 3u : 0u;
        const bool ok = c == 'A' || c == 'C' || c == 'G' || c == 'T';
        const unsigned lo = __ballot_sync(FULL_MASK, code & 1u), hi = __ballot_sync(FULL_MASK, code >> 1), va = __ballot_sync(FULL_MASK, ok);
        if (lane == 0) { s_ix[w] = lo; s_ix[FQ_IX_MAXW + w] = hi; s_ix[2 * FQ_IX_MAXW + w] = va; }
    }
    __syncwarp();
    bool hit = false;
    for (int b0 = 0; b0 < L.n && !hit; b0 += 32) {
        const int b = b0 + lane;
        bool m = false;
        if (b < L.n) {
            const int common = min((int)__ldg(L.lens + b), ilen);
            int diff = 0;
            for (int w = 0; 32 * w < common && diff <= threshold; w++) {
                const uint32_t blo = __ldg(L.words + (size_t)w * L.n + b), bhi = __ldg(L.words + (size_t)(L.W + w) * L.n + b);
                uint32_t x = (s_ix[w] ^ blo) | (s_ix[FQ_IX_MAXW + w] ^ bhi) | ~s_ix[2 * FQ_IX_MAXW + w];
                const int rest = common - 32 * w;
                if (rest < 32) x &= (1u << rest) - 1u;
                diff += __popc(x);
            }
            m = diff <= threshold;
        }
        hit = __any_sync(FULL_MASK, m);
    }
    __syncwarp();                                              /* s_ix is rewritten by the next call */
    return hit;
}

/* flags[i] = whether Filter::filterByIndex removes unit i: one warp per unit.  text2 == NULL: single-end (list 1 only). */
__global__ void __launch_bounds__(32 * FQ_IX_WARPS) fq_index_flags_kernel(const uint8_t* text1, const fq_rec* recs1, const uint8_t* text2, const fq_rec* recs2,
                                                                          long long n, fq_index_list l1, fq_index_list l2, int threshold, uint8_t* flags) {
    __shared__ uint32_t s_ix[FQ_IX_WARPS][3 * FQ_IX_MAXW];
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    for (long long i = (long long)blockIdx.x * FQ_IX_WARPS + w; i < n; i += (long long)gridDim.x * FQ_IX_WARPS) {
        const fq_rec r1 = recs1[i];
        const uint8_t* name1 = text1 + r1.name_off;
        int s, e;
        fq_index_span(name1, (int)(r1.name_len & 0x0FFFFFFFu), true, lane, s, e);
        bool f = fq_index_match(name1, s, e, l1, threshold, s_ix[w], lane);
        if (!f && text2) {
            const fq_rec r2 = recs2[i];
            const uint8_t* name2 = text2 + r2.name_off;
            fq_index_span(name2, (int)(r2.name_len & 0x0FFFFFFFu), false, lane, s, e);
            f = fq_index_match(name2, s, e, l2, threshold, s_ix[w], lane);
        }
        if (lane == 0) flags[i] = f ? 1 : 0;
    }
}
