/*
 * fp_api.cu -- host side of libfastp_b200.so: the C-ABI of include/fastp_b200.h.
 *
 * Context creation precomputes (with the reference's own double expressions) the integer LUTs the
 * kernels use, uploads adapters, sizes the shared-memory tile and the persistent grid.  The
 * fp_process_* entry points enqueue the fused sm_90a kernel (fp_device.cuh); the *_host variants wrap
 * it in a two-stream chunked H2D -> kernel -> D2H pipeline for callers holding host buffers (the
 * reference-side shim of INTEGRATION.md).  No CPU fallback anywhere: without a CUDA device every
 * call fails with FP_E_CUDA.
 */
#include <cuda_runtime.h>
#include <dlfcn.h>
#include <algorithm>
#include <cstdio>
#include <cstring>
#include <cstdlib>
#include <ctime>
#include <chrono>
#include <mutex>
#include <string>
#include <vector>

#include "fastp_b200.h"
#include "fp_device.cuh"
#include "fp_chain2.cuh"
#include "fp_fastq.cuh"
#include "fp_dup.cuh"

static thread_local char g_err[512] = "";
static int set_err(int code, const char* fmt, const char* a = "", const char* b = "") {
    snprintf(g_err, sizeof(g_err), fmt, a, b);
    return code;
}
#define CK(call)                                                                                   \
    do {                                                                                           \
        cudaError_t e_ = (call);                                                                   \
        if (e_ != cudaSuccess) return set_err(FP_E_CUDA, "%s: %s", #call, cudaGetErrorString(e_)); \
    } while (0)

extern "C" const char* fp_last_error(void) { return g_err; }
extern "C" int fp_version(void) { return 100; }

struct EvPair { cudaEvent_t a, b; };

struct fp_ctx {
    int device = 0;
    fp_params p{};
    std::string ad1, ad2;
    std::vector<std::string> fasta;
    fp_dev_params dp{};
    fp_dev_params* d_dp = nullptr;      /* device copy of dp, source of the per-launch constant refresh */
    void* d_cp_sym = nullptr;           /* global address of the __constant__ block */
    cudaEvent_t params_ev = nullptr, last_chain_ev = nullptr;   /* block written by this ctx / its latest chain kernel done */
    bool chain_launched = false;
    fp_counter_layout L{};
    int64_t max_batch = 0;
    int stride = 0, cycles = 0, tile = 0, grid_max = 0, num_sms = 0;
    fp_smem_layout sl{};
    uint32_t smem_base = 1024;        /* shared-window address of dynamic shared memory (probed) */
    cudaStream_t stream[2] = {nullptr, nullptr};
    /* device tables */
    int16_t *d_ovlimit = nullptr, *d_lowq = nullptr, *d_mindiff = nullptr;
    uint8_t* d_adapters = nullptr;
    int32_t *d_fasta_off = nullptr, *d_fasta_len = nullptr;
    uint32_t* d_aplanes = nullptr;
    uint8_t* d_aclean = nullptr;
    /* over-representation analysis (stats.cpp:270-288) */
    std::vector<std::string> overrep[2];
    fp_overrep_side ovr_side[2] = {};
    uint8_t* d_ovr_blob[2] = {nullptr, nullptr};
    int32_t *d_ovr_off[2] = {nullptr, nullptr}, *d_ovr_len[2] = {nullptr, nullptr}, *d_ovr_tidx[2] = {nullptr, nullptr};
    unsigned long long* d_ovr_thash[2] = {nullptr, nullptr};
    uint32_t* d_ovr_bitmap[2] = {nullptr, nullptr};
    unsigned int *d_ovr_blocksum = nullptr, *d_ovr_list = nullptr, *d_ovr_list_n = nullptr;
    unsigned long long* d_ovr_base = nullptr;      /* [2] ping-pong: counted reads seen before this batch */
    int ovr_base_cur = 0;
    int64_t ovr_scratch_n = 0;
    int64_t reads_seen = 0;
    /* adapter-string events (fp_adapter_event) */
    fp_adapter_event* ev_dev = nullptr; uint32_t ev_cap = 0; uint32_t* ev_count = nullptr;      /* device sink (caller's memory) */
    fp_adapter_event* ev_host = nullptr; uint64_t ev_host_cap = 0; uint64_t* ev_host_n = nullptr;  /* host sink of the *_host entry points */
    fp_adapter_event* d_ev[2] = {nullptr, nullptr}; uint32_t* d_nev[2] = {nullptr, nullptr};        /* per chunk slot */
    fp_adapter_event* h_ev[2] = {nullptr, nullptr}; uint32_t* h_nev[2] = {nullptr, nullptr};
    uint32_t ev_chunk_cap = 0;
    int ovr_defer_post = 0;             /* fp_overrep_defer_post: the caller runs fp_overrep_post itself (sharded runs) */
    unsigned long long* d_pass_count = nullptr;
    cudaEvent_t ovr_ev = nullptr;       /* host pipeline: orders the post-filter sampling state between the two chunk streams */
    long long *d_raw = nullptr, *d_fin = nullptr;
    /* host-mode staging (allocated lazily) */
    int64_t chunk = 0;
    uint8_t* d_stage[2][4] = {{nullptr}};      /* seq1 qual1 seq2 qual2 */
    uint16_t* d_stage_len[2][2] = {{nullptr}};
    fp_read_result* d_out[2][2] = {{nullptr}};
    fp_ov_result* d_ov[2] = {nullptr, nullptr};
    fp_patch* d_patch[2] = {nullptr, nullptr};
    unsigned int* d_npatch[2] = {nullptr, nullptr};
    fp_patch* h_patch[4] = {nullptr, nullptr, nullptr, nullptr};      /* host side: 4 rotating buffers (chunk % 4), see process_host */
    unsigned int* h_npatch[4] = {nullptr, nullptr, nullptr, nullptr};
    uint32_t patch_cap = 0;
    uint8_t* d_pk[2][4] = {{nullptr}};          /* packed staging per chunk slot: bases1 qual1 bases2 qual2 */
    fp_npos* d_npos[2] = {nullptr, nullptr};
    size_t pk_cap_b = 0, pk_cap_q = 0, npos_cap = 0;
    /* FP_B_PACK2BIT: pinned host staging of the packing team (4 slots so that it runs two chunks ahead of the copies) */
    uint8_t* h_pkb[4][2] = {{nullptr}};
    fp_npos* h_np[4] = {nullptr, nullptr, nullptr, nullptr};
    size_t h_pkb_cap = 0, h_np_cap = 0;
    int host_threads = 0;                       /* 0 = default_host_threads() */
    cudaEvent_t chunk_done[4] = {nullptr, nullptr, nullptr, nullptr};   /* end of host chunk k's work on its stream, by k % 4 (cudaEventBlockingSync) */
    /* FASTQ codec workspaces (grown on demand) and the buffers of fp_fastq_process_host */
    struct Buf { void* p = nullptr; size_t cap = 0; };
    Buf fq_term, fq_bcnt, fq_agg, fq_bstate, fq_brec, fq_recline, fq_recend, fq_info, fq_bsum;
    Buf fqh_text[2], fqh_seq[2], fqh_qual[2], fqh_len[2], fqh_recs[2], fqh_res[2], fqh_ov, fqh_out[2], fqh_outbuf[2][6], fqh_recend[2];
    unsigned int *fq_hinfo = nullptr, *fq_hinfo_dev = nullptr;      /* mapped pinned control words */
    cudaStream_t fq_stream_out = nullptr;
    cudaEvent_t fq_ev_up = nullptr, fq_ev_out[2] = {nullptr, nullptr};
    /* duplication bloom filter (fp_dup.h) */
    fp_dup_state dup{};
    int dup_level = 0;
    uint64_t* d_dup_primes = nullptr;
    unsigned long long* d_dup_count = nullptr;
    int64_t dup_total = 0;
    const uint8_t* dup_flags = nullptr;     /* fp_set_dup_flags: --dedup flags of the batch the next launch works on */
    int fq_dup_level = 0, fq_dedup = 0;     /* fp_fastq_set_dedup */
    int fq_il_in = 0, fq_il_out = 0;        /* fp_fastq_set_interleaved */
    Buf fq_dupflags;
    Buf dup_pos, dup_keys, dup_vals;
    /* kernel timing */
    std::vector<EvPair> evs;
    std::vector<EvPair> ev_pool;
    double ev_ms = 0.0;
    int64_t ev_n = 0;
};

static void build_luts(const fp_params* p, int stride, std::vector<int16_t>& ov, std::vector<int16_t>& lowq, std::vector<int16_t>& mind) {
    /* the two passFilter tables cover merged reads as well (up to two rows long); the kernel's shared-memory copy takes the first stride + 2 */
    const int maxlen = 2 * stride;
    ov.assign(stride + 2, 0); lowq.assign(maxlen + 2, 0); mind.assign(maxlen + 2, 0);
    const double diffPercentLimit = p->overlap_diff_percent_limit / 100.0;        /* peprocessor.cpp:439 */
    for (int ol = 0; ol <= stride; ol++) {
        int v = std::min(p->overlap_diff_limit, (int)(ol * diffPercentLimit));    /* overlapanalysis.cpp:51 */
        ov[ol] = (int16_t)v;
    }
    for (int rlen = 0; rlen <= maxlen; rlen++) {
        /* lowQualNum > (unqualifiedPercentLimit * rlen / 100.0)   filter.cpp:37 : largest int NOT exceeding the bound */
        double bound = p->unqualified_percent_limit * rlen / 100.0;
        int n = 0;
        while (n <= maxlen && !((double)n > bound)) n++;       /* first n with n > bound */
        lowq[rlen] = (int16_t)(n - 1);
    }
    for (int len = 0; len <= maxlen; len++) {
        /* pass iff (double)diff/(double)(len-1) >= threshold   filter.cpp:65 */
        int d = len + 1;
        if (len > 1) {
            for (int k = 0; k <= len - 1; k++)
                if ((double)k / (double)(len - 1) >= p->complexity_threshold) { d = k; break; }
        }
        mind[len] = (int16_t)d;
    }
}

struct fp_ctx;
struct ParamOwner { std::mutex mu; fp_ctx* owner = nullptr; };
static ParamOwner g_param_owner[64];     /* per device ordinal: which context's parameters the __constant__ block holds */

__global__ void fp_set_params_kernel(uint32_t* dst, const uint32_t* src, int nwords) {
    for (int i = threadIdx.x; i < nwords; i += blockDim.x) dst[i] = src[i];
}

__global__ void fp_probe_smem_base(uint32_t* out) { extern __shared__ uint8_t probe_sm[]; *out = smem_u32(probe_sm); }

static size_t align_up(size_t x, size_t a) { return (x + a - 1) / a * a; }

static size_t smem_layout_for_tile(fp_ctx* c, int T, fp_smem_layout& sl) {
    const int sides = c->p.paired ? 2 : 1;
    const int S = c->stride;
    memset(&sl, 0, sizeof(sl));
    /* ---- tables that live for the whole kernel: sink, LUTs, histograms, delta accumulators, block counters ---- */
    size_t off = 0;
    sl.off_dummy = (int)off; off += 128;
    sl.off_lut = (int)off; off += align_up((size_t)3 * (S + 2) * 2, 16);
    sl.off_delta = (int)off; off += (size_t)sides * (size_t)S * 20 * 4;      /* before the aligned tables: fills what the alignment would waste */
    /* the two histograms are addressed as (field | table address): the 5-mer tables (4 KB per side, counts then signed deltas) must
       start on a 4 KB boundary of the SHARED WINDOW (c->smem_base = window address of dynamic shared memory, probed at fp_ctx_create),
       the quality histograms (2 KB per side + 512 B of deltas) follow */
    off = align_up(off + c->smem_base, 4096) - c->smem_base;
    sl.off_kmer = (int)off; off += (size_t)sides * FP_KMER_BINS * 4;
    sl.off_dkmer = (int)off; off += (size_t)sides * FP_KMER_BINS * 4;       /* signed post-filter deltas, same indexing, same alignment */
    sl.off_qhist = (int)off; off += (size_t)sides * FP_QUAL_BINS * FP_QH_REP * 4;
    sl.off_dqh = (int)off; off += (size_t)sides * FP_QUAL_BINS * 4;
    off = align_up(off, 16);
    sl.off_bc = (int)off; off += sizeof(BlockCounters);
    /* ---- the tile pipeline: mbarrier, cursors, lengths, tile, planes, removal lists, request queue ---- */
    off = align_up(off, 128);
    sl.off_mbar = (int)off; off += 16;
    sl.off_next = (int)off; off += 32;                                     /* queue length, pop cursor, item cursors, correction list length */
    sl.off_len = (int)off; off += (size_t)sides * T * 2;
    sl.off_clean = (int)off; off += (size_t)sides * T;
    off = align_up(off, 128);
    sl.off_tile = (int)off; sl.tile_array_bytes = T * S; off += (size_t)sides * 2 * T * S + 32;   /* + slack for 32-byte plane reads */
    off = align_up(off, 16);
    {   /* removal lists (one per side, padded to 4 entries) + their lengths (4 words), then the same entries in buckets by lo >> 5
           (per-cycle part of phase C) + their lengths; one region, see DeltaSinks */
        const size_t nbk = (size_t)(S + 31) / 32;
        sl.off_rm = (int)off; off += (size_t)sides * (T + 4) * 4 + 16 + sides * nbk * (size_t)(T + 4) * 4 + sides * nbk * 4;
    }
    sl.plane_words = (S + 31) / 32 + 2;
    sl.plane_stride = (5 * sl.plane_words) | 1;                            /* odd: one lane group per row without bank conflicts */
    off = align_up(off, 16);
    sl.off_planes = (int)off; off += (size_t)sides * T * sl.plane_stride * 4;
    off = align_up(off, 16);
    sl.off_queue = (int)off; off += (size_t)sides * T * 2 * 8;
    if (sides == 2) {                                                      /* base correction: work list + per-row masks of corrected positions */
        sl.cm_words = (S + 31) / 32;
        sl.off_corr = (int)off; off += (size_t)FP_CORR_CAP * 4 + 16;                    /* the tile's list + its length */
        sl.off_cm = (int)off; off += (size_t)sides * T * sl.cm_words * 4;
    }
    sl.total = (int)align_up(off, 128);
    return (size_t)sl.total;
}

/* tile size: as large as possible (<= 128 pairs / 256 reads) while one CTA fits an SM's shared memory */
static void make_smem_layout(fp_ctx* c) {
    const int sides = c->p.paired ? 2 : 1;
    const size_t budget = (size_t)227 * 1024;
    int T = sides == 2 ? 128 : 256;                                 /* row indices: 7 bits in the correction list (PE), 8 bits in the removal lists */
    while (T > 16 && smem_layout_for_tile(c, T, c->sl) > budget) T -= 8;
    c->tile = T;
    smem_layout_for_tile(c, T, c->sl);
    /* threads per column of the dense column pass (phase A's dense_tile, phase C's dense_remove): as many as fit in 5/8 of the CTA
       (10 of 16 warps), at least one.  The column pass needs no item and no item needs it, so the warps without columns start the plane /
       histogram items at once and the column warps join them when their rows are done.  With every thread on columns (3 per column at
       2 x 150 bp, 2 at 2 x 250 bp) one warp or none started the items early; on an H100 10 column warps were best for PE and SE at stride
       160 and 8 for PE at stride 256 (DESIGN.md section 9) */
    const int ncols = sides * (c->stride / 2);
    c->sl.col_split = std::max(1, kChainThreads * 5 / 8 / ncols);
}

static int ctx_init(fp_ctx* c, const fp_params* p, int device, int64_t max_batch, int32_t stride, int32_t cycles);
extern "C" void fp_ctx_destroy(fp_ctx* c);

extern "C" int fp_ctx_create(const fp_params* p, int device, int64_t max_batch, int32_t stride, int32_t cycles, fp_ctx** out) {
    if (!p || !out) return set_err(FP_E_INVAL, "null argument");
    if (stride <= 0 || stride % 16 || stride > FP_MAX_STRIDE) return set_err(FP_E_INVAL, "stride must be a multiple of 16 and <= FP_MAX_STRIDE");
    if (cycles <= 0) cycles = stride;
    if (p->allow_gap_overlap_trimming && p->overlap_require < 2) return set_err(FP_E_INVAL, "allow_gap_overlap_trimming needs overlap_require >= 2");
    if (p->insert_size_max < 0 || p->insert_size_max > (1 << 20)) return set_err(FP_E_INVAL, "insert_size_max out of range");
    if ((p->paired ? 2 : 1) * (stride / 2) > 256) return set_err(FP_E_INVAL, "stride too large for the column pass (PE: <= 256, SE: <= 512)");
    if (p->cut_front_window < 1 || p->cut_tail_window < 1 || p->cut_right_window < 1) return set_err(FP_E_INVAL, "cut window must be >= 1");
    int ndev = 0;
    cudaError_t e = cudaGetDeviceCount(&ndev);
    if (e != cudaSuccess || ndev == 0)
        return set_err(FP_E_CUDA, "no CUDA device: fastp_b200 has no CPU fallback (%s)", e != cudaSuccess ? cudaGetErrorString(e) : "device count 0");
    if (device < 0 || device >= ndev) return set_err(FP_E_INVAL, "bad device index");
    CK(cudaSetDevice(device));
    fp_ctx* c = new fp_ctx();
    c->device = device;
    const int rc = ctx_init(c, p, device, max_batch, stride, cycles);
    if (rc != FP_OK) {                                         /* nothing of a partly built context survives (device memory, streams, events) */
        char keep[sizeof(g_err)];
        memcpy(keep, g_err, sizeof(keep));
        fp_ctx_destroy(c);
        memcpy(g_err, keep, sizeof(keep));
        return rc;
    }
    *out = c;
    return FP_OK;
}

static int ctx_init(fp_ctx* c, const fp_params* p, int device, int64_t max_batch, int32_t stride, int32_t cycles) {
    c->p = *p;
    if (p->has_seq_r1 && p->adapter_seq_r1) c->ad1 = p->adapter_seq_r1;
    if (p->has_seq_r2 && p->adapter_seq_r2) c->ad2 = p->adapter_seq_r2;
    for (int i = 0; i < p->n_fasta_adapters; i++) c->fasta.push_back(p->fasta_adapters[i]);
    c->p.adapter_seq_r1 = c->ad1.c_str(); c->p.adapter_seq_r2 = c->ad2.c_str(); c->p.fasta_adapters = nullptr;
    if ((int)c->fasta.size() > FP_MAX_ADAPTERS) { return set_err(FP_E_INVAL, "too many adapters"); }
    for (auto& s : c->fasta) if (s.size() > FP_MAX_ADAPTER_LEN) { return set_err(FP_E_INVAL, "adapter longer than FP_MAX_ADAPTER_LEN"); }
    if (c->ad1.size() > FP_MAX_ADAPTER_LEN || c->ad2.size() > FP_MAX_ADAPTER_LEN) { return set_err(FP_E_INVAL, "adapter longer than FP_MAX_ADAPTER_LEN"); }
    c->max_batch = max_batch; c->stride = stride; c->cycles = cycles;
    if (p->merge_enabled && p->paired && p->overrep_enabled) { return set_err(FP_E_UNSUPPORTED, "merge mode together with over-representation analysis is not built"); }
    if (p->overrep_enabled) {
        if (p->overrep_sampling < 1) { return set_err(FP_E_INVAL, "overrep_sampling must be >= 1"); }
        for (int i = 0; i < p->n_overrep1; i++) c->overrep[0].push_back(p->overrep_seqs1[i]);
        if (p->paired) for (int i = 0; i < p->n_overrep2; i++) c->overrep[1].push_back(p->overrep_seqs2[i]);
    }
    c->p.overrep_seqs1 = nullptr; c->p.overrep_seqs2 = nullptr;
    fp_counter_layout_make_overrep(&c->L, p->paired, cycles, p->insert_size_max, (int)c->overrep[0].size(), p->seq_len1,
                                   (int)c->overrep[1].size(), p->seq_len2);
    {   /* window address of dynamic shared memory (for the aligned histogram tables, see smem_layout_for_tile) */
        uint32_t* d_base = nullptr; uint32_t h_base = 0;
        CK(cudaMalloc(&d_base, 4));
        fp_probe_smem_base<<<1, 1, 16>>>(d_base);
        CK(cudaMemcpy(&h_base, d_base, 4, cudaMemcpyDeviceToHost));
        CK(cudaFree(d_base));
        c->smem_base = h_base;
    }
    make_smem_layout(c);

    cudaDeviceProp prop;
    CK(cudaGetDeviceProperties(&prop, device));
    c->num_sms = prop.multiProcessorCount;
    for (int i = 0; i < 2; i++) CK(cudaStreamCreateWithFlags(&c->stream[i], cudaStreamNonBlocking));
    for (int i = 0; i < 4; i++) CK(cudaEventCreateWithFlags(&c->chunk_done[i], cudaEventBlockingSync | cudaEventDisableTiming));

    /* LUTs */
    std::vector<int16_t> ov, lowq, mind;
    build_luts(p, stride, ov, lowq, mind);
    CK(cudaMalloc(&c->d_ovlimit, ov.size() * 2)); CK(cudaMalloc(&c->d_lowq, lowq.size() * 2)); CK(cudaMalloc(&c->d_mindiff, mind.size() * 2));
    CK(cudaMemcpy(c->d_ovlimit, ov.data(), ov.size() * 2, cudaMemcpyHostToDevice));
    CK(cudaMemcpy(c->d_lowq, lowq.data(), lowq.size() * 2, cudaMemcpyHostToDevice));
    CK(cudaMemcpy(c->d_mindiff, mind.data(), mind.size() * 2, cudaMemcpyHostToDevice));
    /* adapters blob: each adapter at a 16-byte aligned offset, zero padded (+8 readable bytes) */
    std::vector<uint8_t> blob;
    std::vector<int32_t> foff, flen;
    auto put = [&](const std::string& s) { size_t off = blob.size(); blob.insert(blob.end(), s.begin(), s.end()); blob.resize(align_up(blob.size() + 8, 16), 0); return (int)off; };
    fp_dev_params& d = c->dp;
    d.adapter_r1_off = put(c->ad1); d.adapter_r1_len = (int)c->ad1.size();
    d.adapter_r2_off = put(c->ad2); d.adapter_r2_len = (int)c->ad2.size();
    for (auto& s : c->fasta) { foff.push_back(put(s)); flen.push_back((int)s.size()); }
    blob.resize(blob.size() + 16, 0);
    CK(cudaMalloc(&c->d_adapters, blob.size()));
    CK(cudaMemcpy(c->d_adapters, blob.data(), blob.size(), cudaMemcpyHostToDevice));
    if (!foff.empty()) {
        CK(cudaMalloc(&c->d_fasta_off, foff.size() * 4)); CK(cudaMalloc(&c->d_fasta_len, flen.size() * 4));
        CK(cudaMemcpy(c->d_fasta_off, foff.data(), foff.size() * 4, cudaMemcpyHostToDevice));
        CK(cudaMemcpy(c->d_fasta_len, flen.data(), flen.size() * 4, cudaMemcpyHostToDevice));
    }
    {   /* bit planes of every adapter (fp_device.cuh Planes): index 0 = r1, 1 = r2, 2+i = fasta i */
        std::vector<std::string> all = {c->ad1, c->ad2};
        for (auto& s : c->fasta) all.push_back(s);
        std::vector<uint32_t> pl(all.size() * 24, 0);
        std::vector<uint8_t> cl(all.size(), 1);
        for (size_t a = 0; a < all.size(); a++)
            for (size_t k = 0; k < all[a].size(); k++) {
                const unsigned char ch = (unsigned char)all[a][k];
                if (ch == 'N') pl[a * 24 + 16 + (k >> 5)] |= 1u << (k & 31);
                else if (ch == 'A' || ch == 'C' || ch == 'G' || ch == 'T') {
                    const int c2 = (ch >> 1) & 3;
                    if (c2 & 1) pl[a * 24 + 0 + (k >> 5)] |= 1u << (k & 31);
                    if (c2 & 2) pl[a * 24 + 8 + (k >> 5)] |= 1u << (k & 31);
                } else cl[a] = 0;
            }
        CK(cudaMalloc(&c->d_aplanes, pl.size() * 4)); CK(cudaMalloc(&c->d_aclean, cl.size()));
        CK(cudaMemcpy(c->d_aplanes, pl.data(), pl.size() * 4, cudaMemcpyHostToDevice));
        CK(cudaMemcpy(c->d_aclean, cl.data(), cl.size(), cudaMemcpyHostToDevice));
    }
    if (p->overrep_enabled) {
        for (int sd = 0; sd < 2; sd++) {
            const auto& cs = c->overrep[sd];
            fp_overrep_side& S = c->ovr_side[sd];
            S.K = (int)cs.size(); S.eval_len = sd ? p->seq_len2 : p->seq_len1;
            /* a side without candidates has no table: bitmap_mask -1 makes the scan kernel's occupancy copy (words 0 .. mask >> 5)
               empty for it, so the kernel never reads its null bitmap when the other mate has candidates */
            S.bitmap_mask = -1;
            if (S.K == 0) continue;
            std::vector<uint8_t> blob; std::vector<int32_t> off, len;
            for (auto& q : cs) { off.push_back((int32_t)blob.size()); len.push_back((int32_t)q.size()); blob.insert(blob.end(), q.begin(), q.end()); }
            /* sparse table (1/16 full while the occupancy bits fit the kernel's shared-memory copy, never more than 1/4) */
            int tsize = 64;
            while (tsize < 16 * S.K && tsize < FP_OVERREP_BM_BITS) tsize <<= 1;
            while (tsize < 4 * S.K) tsize <<= 1;
            std::vector<unsigned long long> th(tsize, 0); std::vector<int32_t> ti(tsize, -1);
            for (int k = 0; k < S.K; k++) {
                unsigned long long h = 0;
                for (unsigned char ch : cs[k]) h = h * FP_OVERREP_HASH_B + (unsigned long long)(ch + 1);
                if (h == 0) h = 1;
                unsigned int slot = (unsigned int)(h ^ (h >> 32)) & (tsize - 1);
                while (th[slot] != 0) slot = (slot + 1) & (tsize - 1);
                th[slot] = h; ti[slot] = k;
            }
            S.table_mask = tsize - 1;
            const int bm_bits = std::min(tsize, FP_OVERREP_BM_BITS);
            std::vector<uint32_t> bm(bm_bits / 32, 0);
            for (int slot = 0; slot < tsize; slot++) if (th[slot]) { const int bi = slot & (bm_bits - 1); bm[bi >> 5] |= 1u << (bi & 31); }
            S.bitmap_mask = bm_bits - 1;
            const int st5[5] = {10, 20, 40, 100, std::min(150, S.eval_len - 2)};
            for (int i = 0; i < 5; i++) { S.steps[i] = st5[i]; S.bpow[i] = fp_overrep_pow(st5[i]); }
            CK(cudaMalloc(&c->d_ovr_bitmap[sd], bm.size() * 4)); CK(cudaMemcpy(c->d_ovr_bitmap[sd], bm.data(), bm.size() * 4, cudaMemcpyHostToDevice));
            S.bitmap = c->d_ovr_bitmap[sd];
            CK(cudaMalloc(&c->d_ovr_blob[sd], blob.size() + 16)); CK(cudaMemcpy(c->d_ovr_blob[sd], blob.data(), blob.size(), cudaMemcpyHostToDevice));
            CK(cudaMalloc(&c->d_ovr_off[sd], off.size() * 4)); CK(cudaMemcpy(c->d_ovr_off[sd], off.data(), off.size() * 4, cudaMemcpyHostToDevice));
            CK(cudaMalloc(&c->d_ovr_len[sd], len.size() * 4)); CK(cudaMemcpy(c->d_ovr_len[sd], len.data(), len.size() * 4, cudaMemcpyHostToDevice));
            CK(cudaMalloc(&c->d_ovr_thash[sd], (size_t)tsize * 8)); CK(cudaMemcpy(c->d_ovr_thash[sd], th.data(), (size_t)tsize * 8, cudaMemcpyHostToDevice));
            CK(cudaMalloc(&c->d_ovr_tidx[sd], (size_t)tsize * 4)); CK(cudaMemcpy(c->d_ovr_tidx[sd], ti.data(), (size_t)tsize * 4, cudaMemcpyHostToDevice));
            S.blob = c->d_ovr_blob[sd]; S.off = c->d_ovr_off[sd]; S.len = c->d_ovr_len[sd]; S.thash = c->d_ovr_thash[sd]; S.tidx = c->d_ovr_tidx[sd];
        }
        CK(cudaMalloc(&c->d_ovr_base, 16)); CK(cudaMemset(c->d_ovr_base, 0, 16));
        CK(cudaMalloc(&c->d_ovr_list_n, 4));
    }
    CK(cudaMalloc(&c->d_raw, c->L.total * 8)); CK(cudaMalloc(&c->d_fin, c->L.total * 8));
    CK(cudaMemset(c->d_raw, 0, c->L.total * 8)); CK(cudaMemset(c->d_fin, 0, c->L.total * 8));

    d.paired = p->paired; d.thread0 = p->thread0_semantics;
    d.trim_front1 = p->trim_front1; d.trim_tail1 = p->trim_tail1; d.trim_front2 = p->trim_front2; d.trim_tail2 = p->trim_tail2;
    d.max_len1 = p->max_len1; d.max_len2 = p->max_len2;
    d.cut_front = p->cut_front; d.cut_tail = p->cut_tail; d.cut_right = p->cut_right;
    d.cf_w = p->cut_front_window; d.cf_thr = p->cut_front_window * (33 + p->cut_front_quality);      /* filter.cpp:117 */
    d.ct_w = p->cut_tail_window;  d.ct_thr = p->cut_tail_window * (33 + p->cut_tail_quality);        /* filter.cpp:184 */
    d.cr_w = p->cut_right_window; d.cr_thr = p->cut_right_window * (33 + p->cut_right_quality);      /* filter.cpp:151 */
    d.cr_q = 33 + p->cut_right_quality;                                                              /* filter.cpp:159 */
    d.polyg = p->polyg_enabled; d.polyg_min = p->polyg_min_len; d.polyx = p->polyx_enabled; d.polyx_min = p->polyx_min_len;
    d.adapter_enabled = p->adapter_enabled; d.has_r1 = p->has_seq_r1 && !c->ad1.empty() ? 1 : (p->has_seq_r1 ? 1 : 0);
    d.has_r2 = p->has_seq_r2 ? 1 : 0;
    d.n_fasta = (int)c->fasta.size();
    d.fasta_match_req = d.n_fasta > 256 ? 6 : d.n_fasta > 16 ? 5 : 4;                                /* adaptertrimmer.cpp:49-53 */
    d.dimer_max_len = p->dimer_max_len;
    d.merge = p->merge_enabled && p->paired; d.merge_unmerged = p->merge_include_unmerged;
    d.correction = p->correction_enabled; d.ov_require = p->overlap_require; d.allow_gap = p->allow_gap_overlap_trimming; d.ov_diff_limit = p->overlap_diff_limit;
    d.qual_filter = p->qual_filter_enabled; d.qualified_qual = p->qualified_qual & 0xFF; d.n_base_limit = p->n_base_limit; d.avg_qual_req = p->avg_qual_req;
    d.length_filter = p->length_filter_enabled; d.length_required = p->length_required; d.length_limit = p->length_limit;
    d.complexity_filter = p->complexity_filter_enabled;
    d.isize_max = p->insert_size_max;
    d.stride = stride; d.cycles = cycles; d.tile = c->tile; d.n_stats = c->L.n_stats;
    d.lut_ovlimit = c->d_ovlimit; d.lut_lowq = c->d_lowq; d.lut_mindiff = c->d_mindiff;
    d.adapters = c->d_adapters; d.fasta_off = c->d_fasta_off; d.fasta_len = c->d_fasta_len;
    d.adapter_planes = c->d_aplanes; d.adapter_clean = c->d_aclean;
    d.L = c->L;

    /* kernel attributes + persistent grid size */
    int occ = 0;
    {
        const void* fn = p->paired ? (const void*)fp_chain2_kernel<true> : (const void*)fp_chain2_kernel<false>;
        CK(cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, c->sl.total));
        CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, fn, kChainThreads, c->sl.total));
    }
    if (occ < 1) return set_err(FP_E_CUDA, "kernel cannot be resident (shared memory / registers)");
    c->grid_max = occ * c->num_sms;
    if (getenv("FP_TRACE")) fprintf(stderr, "[fastp_b200] chain kernel: tile %d rows, smem %d B, %d CTA/SM, %d threads per column\n", c->tile, c->sl.total, occ, c->sl.col_split);
    return FP_OK;
}

static void fq_free(fp_ctx::Buf& b) { if (b.p) cudaFree(b.p); b.p = nullptr; b.cap = 0; }

static void free_staging(fp_ctx* c) {
    for (int i = 0; i < 2; i++) {
        for (int k = 0; k < 4; k++) { cudaFree(c->d_stage[i][k]); c->d_stage[i][k] = nullptr; }
        for (int k = 0; k < 2; k++) { cudaFree(c->d_stage_len[i][k]); c->d_stage_len[i][k] = nullptr; cudaFree(c->d_out[i][k]); c->d_out[i][k] = nullptr; }
        cudaFree(c->d_ov[i]); c->d_ov[i] = nullptr;
        cudaFree(c->d_patch[i]); c->d_patch[i] = nullptr;
        cudaFree(c->d_npatch[i]); c->d_npatch[i] = nullptr;
        for (int k = 0; k < 4; k++) { cudaFree(c->d_pk[i][k]); c->d_pk[i][k] = nullptr; }
        cudaFree(c->d_npos[i]); c->d_npos[i] = nullptr;
        cudaFree(c->d_ev[i]); c->d_ev[i] = nullptr; cudaFree(c->d_nev[i]); c->d_nev[i] = nullptr;
        if (c->h_ev[i]) cudaFreeHost(c->h_ev[i]); c->h_ev[i] = nullptr;
        if (c->h_nev[i]) cudaFreeHost(c->h_nev[i]); c->h_nev[i] = nullptr;
    }
    for (int i = 0; i < 4; i++) {
        if (c->h_patch[i]) cudaFreeHost(c->h_patch[i]); c->h_patch[i] = nullptr;
        if (c->h_npatch[i]) cudaFreeHost(c->h_npatch[i]); c->h_npatch[i] = nullptr;
        for (int k = 0; k < 2; k++) { if (c->h_pkb[i][k]) cudaFreeHost(c->h_pkb[i][k]); c->h_pkb[i][k] = nullptr; }
        if (c->h_np[i]) cudaFreeHost(c->h_np[i]);
        c->h_np[i] = nullptr;
    }
    c->h_pkb_cap = c->h_np_cap = 0;
    c->chunk = 0; c->pk_cap_b = c->pk_cap_q = c->npos_cap = 0;
}

extern "C" void fp_ctx_destroy(fp_ctx* c) {
    if (!c) return;
    cudaSetDevice(c->device);
    cudaDeviceSynchronize();
    { ParamOwner& po = g_param_owner[c->device & 63]; std::lock_guard<std::mutex> lk(po.mu); if (po.owner == c) po.owner = nullptr; }
    if (c->params_ev) cudaEventDestroy(c->params_ev);
    if (c->last_chain_ev) cudaEventDestroy(c->last_chain_ev);
    free_staging(c);
    {
        fp_ctx::Buf* all[] = {&c->fq_term, &c->fq_bcnt, &c->fq_agg, &c->fq_bstate, &c->fq_brec, &c->fq_recline, &c->fq_recend, &c->fq_info, &c->fq_bsum,
                              &c->fqh_text[0], &c->fqh_text[1], &c->fqh_seq[0], &c->fqh_seq[1], &c->fqh_qual[0], &c->fqh_qual[1], &c->fqh_len[0], &c->fqh_len[1],
                              &c->fqh_recs[0], &c->fqh_recs[1], &c->fqh_res[0], &c->fqh_res[1], &c->fqh_ov, &c->fqh_out[0], &c->fqh_out[1],
                              &c->fqh_recend[0], &c->fqh_recend[1], &c->fq_dupflags};
        for (auto& round : c->fqh_outbuf) for (auto& b : round) fq_free(b);
        if (c->dup.bits) cudaFree(c->dup.bits);
        cudaFree(c->d_dup_primes); cudaFree(c->d_dup_count);
        fq_free(c->dup_pos); fq_free(c->dup_keys); fq_free(c->dup_vals);
        if (c->fq_hinfo) cudaFreeHost(c->fq_hinfo);
        if (c->fq_stream_out) { cudaStreamDestroy(c->fq_stream_out); cudaEventDestroy(c->fq_ev_up); cudaEventDestroy(c->fq_ev_out[0]); cudaEventDestroy(c->fq_ev_out[1]); }
        for (auto* b : all) fq_free(*b);
    }
    cudaFree(c->d_dp);
    cudaFree(c->d_ovlimit); cudaFree(c->d_lowq); cudaFree(c->d_mindiff); cudaFree(c->d_adapters);
    cudaFree(c->d_fasta_off); cudaFree(c->d_fasta_len); cudaFree(c->d_raw); cudaFree(c->d_fin);
    cudaFree(c->d_aplanes); cudaFree(c->d_aclean);
    for (int sd = 0; sd < 2; sd++) { cudaFree(c->d_ovr_blob[sd]); cudaFree(c->d_ovr_off[sd]); cudaFree(c->d_ovr_len[sd]); cudaFree(c->d_ovr_thash[sd]); cudaFree(c->d_ovr_tidx[sd]); cudaFree(c->d_ovr_bitmap[sd]); }
    cudaFree(c->d_ovr_blocksum); cudaFree(c->d_ovr_list); cudaFree(c->d_ovr_list_n); cudaFree(c->d_ovr_base); cudaFree(c->d_pass_count);
    if (c->ovr_ev) cudaEventDestroy(c->ovr_ev);
    for (auto& e : c->evs) { cudaEventDestroy(e.a); cudaEventDestroy(e.b); }
    for (auto& e : c->ev_pool) { cudaEventDestroy(e.a); cudaEventDestroy(e.b); }
    for (int i = 0; i < 2; i++) if (c->stream[i]) cudaStreamDestroy(c->stream[i]);
    for (int i = 0; i < 4; i++) if (c->chunk_done[i]) cudaEventDestroy(c->chunk_done[i]);
    delete c;
}

extern "C" int fp_ctx_layout(const fp_ctx* c, fp_counter_layout* out) {
    if (!c || !out) return set_err(FP_E_INVAL, "null argument");
    *out = c->L;
    return FP_OK;
}

static int drain_events(fp_ctx* c) {
    for (auto& e : c->evs) {
        CK(cudaEventSynchronize(e.b));
        float ms = 0;
        CK(cudaEventElapsedTime(&ms, e.a, e.b));
        c->ev_ms += ms; c->ev_n++;
        c->ev_pool.push_back(e);
    }
    c->evs.clear();
    return FP_OK;
}

/* post-filter over-representation scan of one processed batch (stats.cpp:270-290): rank the counted reads (verdict records),
 * emit the ones whose running count is a multiple of the sampling step, scan their trimmed windows.  host_base == nullptr:
 * continue the ctx's own running count (and advance it); else start from *host_base (sharded runs, fp_overrep_post). */
static int overrep_post_launch(fp_ctx* c, const fp_batch* b, const fp_read_result* out1, const fp_read_result* out2, const int64_t* host_base, cudaStream_t st) {
    const int64_t nblk = (b->n + FP_RANK_ITEMS - 1) / FP_RANK_ITEMS;
    const unsigned int cap = (unsigned int)(b->n / c->p.overrep_sampling + 64);
    if (b->n > c->ovr_scratch_n) {
        CK(cudaStreamSynchronize(st));
        cudaFree(c->d_ovr_blocksum); cudaFree(c->d_ovr_list);
        CK(cudaMalloc(&c->d_ovr_blocksum, (size_t)(nblk + 1) * 4)); CK(cudaMalloc(&c->d_ovr_list, (size_t)cap * 4));
        c->ovr_scratch_n = b->n;
    }
    unsigned long long* base_cur = c->d_ovr_base + c->ovr_base_cur; unsigned long long* base_next = c->d_ovr_base + (c->ovr_base_cur ^ 1);
    if (host_base) {
        const unsigned long long v = (unsigned long long)*host_base;
        CK(cudaMemcpyAsync(base_cur, &v, 8, cudaMemcpyHostToDevice, st));   /* pageable source: staged by the runtime before the call returns */
    }
    fp_overrep_args oa;
    memset(&oa, 0, sizeof(oa));
    oa.b = *b; oa.side[0] = c->ovr_side[0]; oa.side[1] = c->ovr_side[1];
    oa.counters = reinterpret_cast<unsigned long long*>(c->d_raw); oa.L = c->L;
    oa.sides = c->p.paired ? 2 : 1; oa.sampling = c->p.overrep_sampling;
    CK(cudaMemsetAsync(c->d_ovr_list_n, 0, 4, st));
    fp_overrep_blocksum_kernel<<<(unsigned)nblk, 256, 0, st>>>(out1, b->n, c->d_ovr_blocksum);
    fp_overrep_scan_kernel<<<1, 32, 0, st>>>(c->d_ovr_blocksum, (int)nblk, base_cur, base_next);
    fp_overrep_emit_kernel<<<(unsigned)nblk, 256, 0, st>>>(out1, b->n, c->d_ovr_blocksum, base_cur, c->p.overrep_sampling, c->d_ovr_list, c->d_ovr_list_n, cap);
    oa.post = 1; oa.res[0] = out1; oa.res[1] = out2; oa.list = c->d_ovr_list; oa.list_n = c->d_ovr_list_n;
    const long long warps = (long long)cap * oa.sides;
    fp_overrep_kernel<<<(unsigned)((warps + 7) / 8), 256, 0, st>>>(oa);
    CK(cudaGetLastError());
    c->ovr_base_cur ^= 1;
    return FP_OK;
}

static int launch_chain(fp_ctx* c, const fp_batch* b, fp_read_result* out1, fp_read_result* out2, fp_ov_result* ov,
                        fp_patch* patches, uint32_t patch_cap, uint32_t* n_patches, cudaStream_t st) {
    if (b->n == 0) return FP_OK;
    if (b->stride != c->stride) return set_err(FP_E_INVAL, "batch stride differs from the ctx stride");
    if (b->n > (int64_t)1 << 31) return set_err(FP_E_TOOLARGE, "batch larger than 2^31 (split it)");
    auto mis = [](const void* q) { return ((uintptr_t)q & 15) != 0; };
    if (mis(b->seq1) || mis(b->qual1) || (c->p.paired && (mis(b->seq2) || mis(b->qual2)))) return set_err(FP_E_INVAL, "seq/qual pointers must be 16-byte aligned");
    fp_launch_args a;
    memset(&a, 0, sizeof(a));
    a.b = *b; a.out1 = out1; a.out2 = out2; a.ov = ov;
    a.sink.patches = patches; a.sink.cap = patches ? patch_cap : 0; a.sink.count = n_patches;
    a.is_dup = c->dup_flags;
    a.events.events = c->ev_dev; a.events.cap = c->ev_dev ? c->ev_cap : 0; a.events.count = c->ev_count;
    a.counters = reinterpret_cast<unsigned long long*>(c->d_raw);
    a.n_tiles = (b->n + c->tile - 1) / c->tile;
    a.sl = c->sl;
    int grid = (int)std::min<long long>(a.n_tiles, c->grid_max);
    /* The operator parameters live in ONE __constant__ block per device, owned by the context that launched last.  A launch by the owner
       costs nothing; a launch by another context first waits -- on the device, in its own stream -- for the owner's last chain kernel
       (the only reader of the block), then rewrites the block from its device copy with a small kernel (stream-ordered, no copy engine:
       a cudaMemcpyToSymbolAsync would queue behind bulk transfers).  Contexts with different parameters therefore alternate correctly
       on one device; they just do not overlap each other's chain kernels. */
    if (!c->d_dp) {
        CK(cudaMalloc(&c->d_dp, sizeof(fp_dev_params)));
        CK(cudaMemcpy(c->d_dp, &c->dp, sizeof(fp_dev_params), cudaMemcpyHostToDevice));
        CK(cudaGetSymbolAddress((void**)&c->d_cp_sym, c_p));
        CK(cudaEventCreateWithFlags(&c->params_ev, cudaEventDisableTiming));
        CK(cudaEventCreateWithFlags(&c->last_chain_ev, cudaEventDisableTiming));
    }
    ParamOwner& po = g_param_owner[c->device & 63];
    std::unique_lock<std::mutex> plk(po.mu);
    if (po.owner != c) {
        if (po.owner && po.owner->last_chain_ev && po.owner->chain_launched) CK(cudaStreamWaitEvent(st, po.owner->last_chain_ev, 0));
        fp_set_params_kernel<<<1, 128, 0, st>>>(reinterpret_cast<uint32_t*>(c->d_cp_sym), reinterpret_cast<const uint32_t*>(c->d_dp), (int)(sizeof(fp_dev_params) / 4));
        CK(cudaEventRecord(c->params_ev, st));
        po.owner = c;
    } else {
        CK(cudaStreamWaitEvent(st, c->params_ev, 0));          /* the block was written in another of this context's streams */
    }
    fp_overrep_args oa;
    const bool ovr = c->p.overrep_enabled && (c->ovr_side[0].K > 0 || c->ovr_side[1].K > 0);
    if (ovr) {
        memset(&oa, 0, sizeof(oa));
        oa.b = *b; oa.side[0] = c->ovr_side[0]; oa.side[1] = c->ovr_side[1];
        oa.counters = reinterpret_cast<unsigned long long*>(c->d_raw); oa.L = c->L;
        oa.sides = c->p.paired ? 2 : 1; oa.sampling = c->p.overrep_sampling;
        /* pre-filter stats: the ORIGINAL rows, i.e. before the chain kernel may correct bases in place */
        oa.post = 0; oa.first_index = (b->flags & FP_B_INDEXED) ? b->first_read_index : c->reads_seen;
        const long long units = (b->n + oa.sampling - 1) / oa.sampling + 1;
        const long long warps = units * oa.sides;
        fp_overrep_kernel<<<(unsigned)((warps + 7) / 8), 256, 0, st>>>(oa);
        CK(cudaGetLastError());
    }
    EvPair ev;
    if (!c->ev_pool.empty()) { ev = c->ev_pool.back(); c->ev_pool.pop_back(); }
    else { CK(cudaEventCreate(&ev.a)); CK(cudaEventCreate(&ev.b)); }
    if (c->evs.size() > 4096) { int rc = drain_events(c); if (rc) return rc; }
    CK(cudaEventRecord(ev.a, st));
    {
        void* kargs[] = {(void*)&a};
        const void* fn = c->p.paired ? (const void*)fp_chain2_kernel<true> : (const void*)fp_chain2_kernel<false>;
        CK(cudaLaunchKernel(fn, dim3(grid), dim3(kChainThreads), kargs, (size_t)c->sl.total, st));
    }
    CK(cudaEventRecord(ev.b, st));
    CK(cudaEventRecord(c->last_chain_ev, st));
    c->chain_launched = true;
    plk.unlock();
    c->evs.push_back(ev);
    CK(cudaGetLastError());
    if (ovr) {
        if (!c->ovr_defer_post) {
            int rc = overrep_post_launch(c, b, out1, out2, nullptr, st);
            if (rc) return rc;
        }
        c->reads_seen = ((b->flags & FP_B_INDEXED) ? b->first_read_index : c->reads_seen) + b->n;
    }
    return FP_OK;
}

extern "C" int fp_process_se(fp_ctx* c, const fp_batch* b, fp_read_result* out1, void* stream) {
    if (!c || !b || !out1) return set_err(FP_E_INVAL, "null argument");
    if (c->p.paired) return set_err(FP_E_INVAL, "ctx was created for paired-end data");
    CK(cudaSetDevice(c->device));
    return launch_chain(c, b, out1, nullptr, nullptr, nullptr, 0, nullptr, stream ? (cudaStream_t)stream : c->stream[0]);
}

extern "C" int fp_process_pe(fp_ctx* c, const fp_batch* b, fp_read_result* out1, fp_read_result* out2, fp_ov_result* ov,
                             fp_patch* patches, uint32_t patch_cap, uint32_t* n_patches, void* stream) {
    if (!c || !b || !out1 || !out2) return set_err(FP_E_INVAL, "null argument");
    if (!c->p.paired) return set_err(FP_E_INVAL, "ctx was created for single-end data");
    CK(cudaSetDevice(c->device));
    return launch_chain(c, b, out1, out2, ov, patches, patch_cap, n_patches, stream ? (cudaStream_t)stream : c->stream[0]);
}

/* ---------------- undo of a pass's base corrections / sharded over-representation sampling ---------------- */
__global__ void fp_patch_undo_kernel(fp_batch b, const fp_patch* __restrict__ patches, const uint32_t* __restrict__ n_patches, uint32_t cap) {
    const uint32_t n = min(*n_patches, cap);
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const fp_patch pt = patches[i];
        const size_t o = (size_t)pt.pair * (size_t)b.stride + pt.pos;
        (pt.which ? b.seq2 : b.seq1)[o] = pt.old_base;
        (pt.which ? b.qual2 : b.qual1)[o] = pt.old_qual;
    }
}

extern "C" int fp_patches_undo(fp_ctx* c, const fp_batch* b, const fp_patch* patches, const uint32_t* n_patches, uint32_t patch_cap, void* stream) {
    if (!c || !b || !patches || !n_patches) return set_err(FP_E_INVAL, "null argument");
    if (!c->p.paired) return set_err(FP_E_INVAL, "base correction is a paired-end operator");
    CK(cudaSetDevice(c->device));
    cudaStream_t st = stream ? (cudaStream_t)stream : c->stream[0];
    if (patch_cap == 0) return FP_OK;
    const unsigned blocks = (unsigned)std::min<uint64_t>(((uint64_t)patch_cap + 255) / 256, (uint64_t)c->num_sms * 8);
    fp_patch_undo_kernel<<<blocks, 256, 0, st>>>(*b, patches, n_patches, patch_cap);
    CK(cudaGetLastError());
    return FP_OK;
}

__global__ void fp_pass_count_kernel(const fp_read_result* __restrict__ res, long long n, unsigned long long* out) {
    unsigned int c = 0;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) c += (res[i].pair_verdict == FP_PASS_FILTER);
    #pragma unroll
    for (int o = 16; o > 0; o >>= 1) c += __shfl_xor_sync(FULL_MASK, c, o);
    if ((threadIdx.x & 31) == 0 && c) atomicAdd(out, (unsigned long long)c);
}

extern "C" int fp_overrep_defer_post(fp_ctx* c, int32_t defer) {
    if (!c) return set_err(FP_E_INVAL, "null argument");
    c->ovr_defer_post = defer ? 1 : 0;
    return FP_OK;
}

extern "C" int fp_pass_count(fp_ctx* c, const fp_read_result* out1, int64_t n, int64_t* count, void* stream) {
    if (!c || !count || (n > 0 && !out1)) return set_err(FP_E_INVAL, "null argument");
    CK(cudaSetDevice(c->device));
    cudaStream_t st = stream ? (cudaStream_t)stream : c->stream[0];
    if (!c->d_pass_count) CK(cudaMalloc(&c->d_pass_count, 8));
    CK(cudaMemsetAsync(c->d_pass_count, 0, 8, st));
    if (n > 0) {
        const unsigned blocks = (unsigned)std::min<int64_t>((n + 255) / 256, (int64_t)c->num_sms * 16);
        fp_pass_count_kernel<<<blocks, 256, 0, st>>>(out1, n, c->d_pass_count);
        CK(cudaGetLastError());
    }
    unsigned long long v = 0;
    CK(cudaMemcpyAsync(&v, c->d_pass_count, 8, cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    *count = (int64_t)v;
    return FP_OK;
}

extern "C" int fp_overrep_post(fp_ctx* c, const fp_batch* b, const fp_read_result* out1, const fp_read_result* out2, int64_t pass_base, void* stream) {
    if (!c || !b || !out1) return set_err(FP_E_INVAL, "null argument");
    if (c->p.paired && !out2) return set_err(FP_E_INVAL, "paired ctx needs the second side's records");
    if (pass_base < 0) return set_err(FP_E_INVAL, "pass_base must be >= 0");
    CK(cudaSetDevice(c->device));
    if (!(c->p.overrep_enabled && (c->ovr_side[0].K > 0 || c->ovr_side[1].K > 0)) || b->n == 0) return FP_OK;
    if (b->stride != c->stride) return set_err(FP_E_INVAL, "batch stride differs from the ctx stride");
    return overrep_post_launch(c, b, out1, out2, &pass_base, stream ? (cudaStream_t)stream : c->stream[0]);
}

extern "C" int fp_set_event_sink(fp_ctx* c, fp_adapter_event* d_events, uint32_t cap, uint32_t* d_count) {
    if (!c) return set_err(FP_E_INVAL, "null argument");
    if (d_count && cap > 0 && !d_events) return set_err(FP_E_INVAL, "event list missing");
    c->ev_dev = d_count ? d_events : nullptr; c->ev_cap = d_count ? cap : 0; c->ev_count = d_count;
    return FP_OK;
}

extern "C" int fp_set_host_event_sink(fp_ctx* c, fp_adapter_event* h_events, uint64_t cap, uint64_t* n_events) {
    if (!c) return set_err(FP_E_INVAL, "null argument");
    if (n_events && cap > 0 && !h_events) return set_err(FP_E_INVAL, "event list missing");
    c->ev_host = n_events ? h_events : nullptr; c->ev_host_cap = n_events ? cap : 0; c->ev_host_n = n_events;
    return FP_OK;
}

/* ---------------- packed host rows (fp_packed_batch) ---------------- */
/* one thread per (read, 16 bases): 4 packed bytes -> 16 ASCII bases, 16 qualities re-pitched; zero fill beyond the read */
__global__ void fp_unpack_kernel(const uint8_t* __restrict__ pb, const uint8_t* __restrict__ pq, const uint16_t* __restrict__ len, long long n,
                                 int pitch_b, int pitch_q, int stride, uint8_t* __restrict__ seq, uint8_t* __restrict__ qual) {
    const int gpr = stride >> 4;                                           /* 16-byte groups per row */
    const long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x;
    if (t >= n * gpr) return;
    const long long r = t / gpr; const int g = (int)(t - r * gpr);
    const int L = min((int)len[r], stride);
    const uint8_t* b = pb + r * pitch_b + g * 4; const uint8_t* q = pq + r * pitch_q + g * 16;
    uint32_t so[4], qo[4];
    #pragma unroll
    for (int w = 0; w < 4; w++) {
        const int p0 = g * 16 + w * 4;
        uint32_t sv = 0, qv = 0;
        if (p0 < L) {
            const uint32_t c = b[w];
            #pragma unroll
            for (int k = 0; k < 4; k++)
                if (p0 + k < L) { sv |= ((0x47544341u >> (8 * ((c >> (2 * k)) & 3u))) & 0xFFu) << (8 * k); qv |= (uint32_t)q[w * 4 + k] << (8 * k); }
        }
        so[w] = sv; qo[w] = qv;
    }
    *reinterpret_cast<uint4*>(seq + r * stride + g * 16) = make_uint4(so[0], so[1], so[2], so[3]);
    *reinterpret_cast<uint4*>(qual + r * stride + g * 16) = make_uint4(qo[0], qo[1], qo[2], qo[3]);
}
/* host rows at a tighter pitch than the device stride (no padding over PCIe): one thread per (read, 16 output bytes) */
__global__ void fp_repitch_kernel(const uint8_t* __restrict__ in, const uint16_t* __restrict__ len, long long n, int pitch, int stride, uint8_t* __restrict__ out) {
    const int gpr = stride >> 4;
    const long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x;
    if (t >= n * gpr) return;
    const long long r = t / gpr; const int g = (int)(t - r * gpr);
    const int L = min((int)len[r], min(stride, pitch));
    const uint8_t* s = in + r * pitch + g * 16;
    uint32_t o[4];
    #pragma unroll
    for (int w = 0; w < 4; w++) {
        uint32_t v = 0;
        #pragma unroll
        for (int k = 0; k < 4; k++) { const int p = g * 16 + w * 4 + k; if (p < L) v |= (uint32_t)s[w * 4 + k] << (8 * k); }
        o[w] = v;
    }
    *reinterpret_cast<uint4*>(out + r * stride + g * 16) = make_uint4(o[0], o[1], o[2], o[3]);
}
__global__ void fp_unpack_n_kernel(const fp_npos* __restrict__ np, long long cnt, long long unit0, int stride, uint8_t* seq1, uint8_t* seq2) {
    const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
    if (i >= cnt) return;
    const fp_npos e = np[i];
    (e.which ? seq2 : seq1)[((long long)e.unit - unit0) * stride + e.pos] = 'N';
}

#include <thread>
#include <atomic>
#include <memory>
#include <mutex>
#include <condition_variable>
#include <sched.h>
#include "fp_hostpack.h"

/* CPUs this process may really use: the affinity mask, cut by a cgroup CPU quota (a container with 16 CPUs of a 128-core box) */
static int usable_cpus() {
    int n = (int)std::thread::hardware_concurrency();
    cpu_set_t set;
    if (sched_getaffinity(0, sizeof(set), &set) == 0) n = CPU_COUNT(&set);
    if (FILE* f = fopen("/sys/fs/cgroup/cpu.max", "r")) {
        char q[64]; long long period = 0;
        if (fscanf(f, "%63s %lld", q, &period) == 2 && strcmp(q, "max") != 0 && period > 0) n = std::min<long long>(n, std::max<long long>(1, atoll(q) / period));
        fclose(f);
    } else {
        long long quota = -1, period = 0;
        if (FILE* g = fopen("/sys/fs/cgroup/cpu/cpu.cfs_quota_us", "r")) { if (fscanf(g, "%lld", &quota) != 1) quota = -1; fclose(g); }
        if (FILE* g = fopen("/sys/fs/cgroup/cpu/cpu.cfs_period_us", "r")) { if (fscanf(g, "%lld", &period) != 1) period = 0; fclose(g); }
        if (quota > 0 && period > 0) n = std::min<long long>(n, std::max<long long>(1, quota / period));
    }
    return std::max(n, 1);
}
static int default_host_threads() { return std::min(std::max(usable_cpus() - 1, 1), 32); }

extern "C" int fp_set_host_threads(fp_ctx* c, int threads) {
    if (!c || threads < 0) return set_err(FP_E_INVAL, "bad argument");
    c->host_threads = threads;
    return FP_OK;
}

extern "C" int fp_host_pack_rows(const fp_batch* rows, int paired, fp_packed_batch* out, int threads) {
    if (!rows || !out || !out->bases1 || !out->qual1 || !out->len1 || (paired && (!out->bases2 || !out->qual2 || !out->len2))) return set_err(FP_E_INVAL, "null argument");
    if (rows->n >= ((int64_t)1 << 32)) return set_err(FP_E_TOOLARGE, "batch larger than 2^32");
    const int64_t n = rows->n; const int S = rows->stride, pb = out->pitch_b, pq = out->pitch_q;
    if (threads < 1) threads = 1;
    threads = (int)std::min<int64_t>(threads, std::max<int64_t>(1, n / 4096));
    std::vector<std::vector<fp_npos>> nl(threads);
    std::vector<int> bad(threads, 0);
    auto work = [&](int t) {
        const int64_t lo = n * t / threads, hi = n * (t + 1) / threads;
        for (int64_t r = lo; r < hi; r++)                                  /* read 1 then read 2 of a unit: the list comes out sorted by unit */
            for (int sd = 0; sd < (paired ? 2 : 1); sd++) {
                const uint8_t* seq = sd ? rows->seq2 : rows->seq1; const uint8_t* qual = sd ? rows->qual2 : rows->qual1; const uint16_t* len = sd ? rows->len2 : rows->len1;
                uint8_t* ob = sd ? out->bases2 : out->bases1; uint8_t* oq = sd ? out->qual2 : out->qual1; uint16_t* ol = sd ? out->len2 : out->len1;
                const int L = len[r];
                if ((L + 3) / 4 > pb || L > pq || L > S) { bad[t] = 2; return; }
                if (fp_pack_bases_row(seq + r * S, L, ob + r * pb, (uint32_t)r, sd, nl[t])) { bad[t] = 1; return; }
                memcpy(oq + r * pq, qual + r * S, L);
                ol[r] = (uint16_t)L;
            }
    };
    std::vector<std::thread> th;
    for (int t = 1; t < threads; t++) th.emplace_back(work, t);
    work(0);
    for (auto& x : th) x.join();
    for (int t = 0; t < threads; t++) {
        if (bad[t] == 1) return set_err(FP_E_UNSUPPORTED, "a base outside {A,C,G,T,N}: not representable in packed rows");
        if (bad[t] == 2) return set_err(FP_E_INVAL, "a read is longer than the packed pitch");
    }
    /* exception list sorted by unit: every thread's entries come side by side (read1 then read2 of its range), ranges are in order */
    int64_t total = 0;
    for (auto& v : nl) total += (int64_t)v.size();
    out->n_npos = total;
    if (total > out->npos_cap) return set_err(FP_E_TOOLARGE, "N exception list too small (n_npos holds the size needed)");
    int64_t o = 0;
    for (auto& v : nl) {
        if (!v.empty()) memcpy(out->npos + o, v.data(), v.size() * sizeof(fp_npos));
        o += (int64_t)v.size();
    }
    out->n = n; out->flags = rows->flags; out->first_read_index = rows->first_read_index;
    return FP_OK;
}

/* ---------------- host-buffer pipeline ---------------- */
static int ensure_staging(fp_ctx* c) {
    if (c->chunk) return FP_OK;
    const int sides = c->p.paired ? 2 : 1;
    int64_t chunk = std::min<int64_t>(std::max<int64_t>(c->max_batch, 1), (int64_t)1 << 18);
    chunk = (chunk + c->tile - 1) / c->tile * c->tile;
    c->chunk = chunk;
    c->patch_cap = (uint32_t)std::min<int64_t>(chunk * 2 + 1024, (int64_t)1 << 22);
    for (int i = 0; i < 2; i++) {
        for (int k = 0; k < 2 * sides; k++) CK(cudaMalloc(&c->d_stage[i][k], (size_t)chunk * c->stride + 64));
        for (int k = 0; k < sides; k++) { CK(cudaMalloc(&c->d_stage_len[i][k], (size_t)chunk * 2)); CK(cudaMalloc(&c->d_out[i][k], (size_t)chunk * sizeof(fp_read_result))); }
        if (c->p.paired) {
            CK(cudaMalloc(&c->d_ov[i], (size_t)chunk * sizeof(fp_ov_result)));
            CK(cudaMalloc(&c->d_patch[i], (size_t)c->patch_cap * sizeof(fp_patch)));
            CK(cudaMalloc(&c->d_npatch[i], 4));
        }
    }
    if (c->p.paired)
        for (int i = 0; i < 4; i++) {
            CK(cudaMallocHost(&c->h_patch[i], (size_t)c->patch_cap * sizeof(fp_patch)));
            CK(cudaMallocHost(&c->h_npatch[i], 4));
        }
    return FP_OK;
}

/* the whole patch buffer of a chunk rides along with its results (about 2 % of the chunk's input bytes): no second round trip for its count */

static int process_host(fp_ctx* c, const fp_batch* b, fp_read_result* out1, fp_read_result* out2, fp_ov_result* ov,
                        fp_patch* hp_out = nullptr, uint64_t hp_cap = 0, uint64_t* hp_n = nullptr, const fp_packed_batch* pk = nullptr) {
    if (hp_n) *hp_n = 0;
    /* the chain indexes the flags by the unit's index in its LAUNCH, and a host batch is launched chunk by chunk */
    if (c->dup_flags) return set_err(FP_E_INVAL, "duplicate flags are set (fp_set_dup_flags): they belong to one fp_process_se / _pe launch, not to a host batch");
    CK(cudaSetDevice(c->device));
    int rc = ensure_staging(c);
    if (rc) return rc;
    /* host rows may be tighter than the device stride (pitch = read length: no padding bytes over PCIe); they are re-pitched in HBM */
    const int HP = b->stride;
    if (HP > c->stride || HP <= 0) return set_err(FP_E_INVAL, "host row pitch must be in (0, ctx stride]");
    const bool packfly = !pk && (b->flags & FP_B_PACK2BIT) != 0;
    const bool repitch = !pk && !packfly && HP != c->stride;
    const int PB = ((((HP + 3) >> 2) + 3) & ~3);                 /* packed bases of one row, FP_B_PACK2BIT */
    const int NS = 4;                                          /* host staging slots of the packing team */
    if (packfly) {
        const size_t nb = (size_t)c->chunk * PB + 64, nq = (size_t)c->chunk * HP + 64;
        if (nb > c->pk_cap_b || nq > c->pk_cap_q) {
            CK(cudaDeviceSynchronize());
            for (int i = 0; i < 2; i++)
                for (int k = 0; k < (c->p.paired ? 4 : 2); k++) { cudaFree(c->d_pk[i][k]); c->d_pk[i][k] = nullptr; CK(cudaMalloc(&c->d_pk[i][k], (k & 1) ? nq : nb)); }
            c->pk_cap_b = nb; c->pk_cap_q = nq;
        }
        if (nb > c->h_pkb_cap) {
            for (int i = 0; i < NS; i++)
                for (int k = 0; k < (c->p.paired ? 2 : 1); k++) { if (c->h_pkb[i][k]) cudaFreeHost(c->h_pkb[i][k]); c->h_pkb[i][k] = nullptr; CK(cudaMallocHost(&c->h_pkb[i][k], nb)); }
            c->h_pkb_cap = nb;
        }
    }
    if (repitch) {
        const size_t nb = (size_t)c->chunk * HP + 64;
        if (nb > c->pk_cap_b || nb > c->pk_cap_q) {
            CK(cudaDeviceSynchronize());
            for (int i = 0; i < 2; i++)
                for (int k = 0; k < (c->p.paired ? 4 : 2); k++) { cudaFree(c->d_pk[i][k]); c->d_pk[i][k] = nullptr; CK(cudaMalloc(&c->d_pk[i][k], nb)); }
            c->pk_cap_b = c->pk_cap_q = nb;
        }
    }
    if (pk) {                                                  /* packed input: staging for one chunk of packed rows + its N exceptions */
        if (pk->pitch_b <= 0 || pk->pitch_q <= 0) return set_err(FP_E_INVAL, "bad packed pitch");
        const size_t nb = (size_t)c->chunk * pk->pitch_b + 64, nq = (size_t)c->chunk * pk->pitch_q + 64;
        if (nb > c->pk_cap_b || nq > c->pk_cap_q) {
            CK(cudaDeviceSynchronize());
            for (int i = 0; i < 2; i++)
                for (int k = 0; k < (c->p.paired ? 4 : 2); k++) { cudaFree(c->d_pk[i][k]); CK(cudaMalloc(&c->d_pk[i][k], (k & 1) ? nq : nb)); }
            c->pk_cap_b = nb; c->pk_cap_q = nq;
        }
    }
    const bool pe = c->p.paired;
    const int S = c->stride;
    const int64_t n = b->n, CH = c->chunk;
    const int64_t nchunks = (n + CH - 1) / CH;
    struct Pending { int64_t lo, cnt; bool active; } pend[4] = {{0, 0, false}, {0, 0, false}, {0, 0, false}, {0, 0, false}};   /* by chunk % 4 */
    const bool want_ev = c->ev_host_n != nullptr;
    if (want_ev) {
        *c->ev_host_n = 0;
        if (!c->d_ev[0]) {
            /* a pair gives at most 2 events (trimByOverlapAnalysis, or trimBySequence on each read) + 1 per fasta adapter and read; a read
               1 + 1 per fasta adapter.  Past 2^24 entries (a full chunk with more than 30 fasta adapters PE, 62 SE) a chunk could still
               overflow: finish() fails then */
            const int64_t per_unit = pe ? 2 + 2 * (int64_t)c->p.n_fasta_adapters : 1 + (int64_t)c->p.n_fasta_adapters;
            c->ev_chunk_cap = (uint32_t)std::min<int64_t>(CH * per_unit + 1024, (int64_t)1 << 24);
            for (int i = 0; i < 2; i++) {
                CK(cudaMalloc(&c->d_ev[i], (size_t)c->ev_chunk_cap * sizeof(fp_adapter_event))); CK(cudaMalloc(&c->d_nev[i], 4));
                CK(cudaMallocHost(&c->h_ev[i], (size_t)c->ev_chunk_cap * sizeof(fp_adapter_event))); CK(cudaMallocHost(&c->h_nev[i], 4));
            }
        }
    }
    /* the device sink of fp_set_event_sink (if any) is put back when this call returns */
    fp_adapter_event* const saved_dev = c->ev_dev; const uint32_t saved_cap = c->ev_cap; uint32_t* const saved_cnt = c->ev_count;
    struct Restore { fp_ctx* c; fp_adapter_event* d; uint32_t cap; uint32_t* n; ~Restore() { c->ev_dev = d; c->ev_cap = cap; c->ev_count = n; } } restore{c, saved_dev, saved_cap, saved_cnt};
    if (!want_ev) { c->ev_dev = nullptr; c->ev_cap = 0; c->ev_count = nullptr; }
    /* a chunk that fails in finish() returns early: leave no copy into the caller's buffers in flight behind the return */
    struct Drain { fp_ctx* c; ~Drain() { cudaStreamSynchronize(c->stream[0]); cudaStreamSynchronize(c->stream[1]); } } drain{c};
    /* finish(k): host side of chunk k.  Device buffers belong to slot k & 1, the host patch buffers and `pend` to k % 4: the device slot
       is handed to chunk k + 2 as soon as the chunk's event has fired, while its patches are still being written back here. */
    auto finish = [&](int64_t k) -> int {
        const int slot = (int)(k & 1), hs = (int)(k & 3);
        if (!pend[hs].active) return FP_OK;
        CK(cudaEventSynchronize(c->chunk_done[hs]));             /* blocking-sync event: the waiting thread sleeps instead of spinning.  One event per
                                                                    chunk in flight on the HOST side (k % 4): the slot's next chunk records its own */
        if (want_ev) {
            const uint32_t ne = *c->h_nev[slot];
            /* the kernel dropped what did not fit: the caller's list would have a hole in the middle */
            if (ne > c->ev_chunk_cap) return set_err(FP_E_TOOLARGE, "adapter events of one host chunk exceed its event buffer (too many fasta adapters)");
            if (ne > 0) CK(cudaMemcpy(c->h_ev[slot], c->d_ev[slot], (size_t)ne * sizeof(fp_adapter_event), cudaMemcpyDeviceToHost));
            for (uint32_t i = 0; i < ne; i++) {
                if (*c->ev_host_n < c->ev_host_cap) { c->ev_host[*c->ev_host_n] = c->h_ev[slot][i]; c->ev_host[*c->ev_host_n].unit = (uint32_t)(pend[hs].lo + c->h_ev[slot][i].unit); }
                (*c->ev_host_n)++;
            }
        }
        if (pe && c->p.correction_enabled) {
            uint32_t np = *c->h_npatch[hs];
            const int64_t lo = pend[hs].lo;
            if (np <= c->patch_cap) {
                /* the write-back touches two random cache lines per correction: memory-latency bound (16 ns per patch on one core, 3 ms per
                   chunk -- more than the chunk's transfer).  The lines of the patch 24 entries ahead are requested while this one is
                   applied, and a large list is split over four threads (no two patches touch the same byte). */
                const fp_patch* const P = c->h_patch[hs];
                if (!pk) {
                    auto apply_range = [&](uint32_t a0, uint32_t a1) {
                        for (uint32_t i = a0; i < a1; i++) {
                            const fp_patch& pt = P[i];
                            if (i + 24 < a1) {
                                const fp_patch& nx = P[i + 24];
                                __builtin_prefetch((nx.which ? b->seq2 : b->seq1) + (lo + nx.pair) * HP + nx.pos, 1, 0);
                                __builtin_prefetch((nx.which ? b->qual2 : b->qual1) + (lo + nx.pair) * HP + nx.pos, 1, 0);
                            }
                            uint8_t* sq = (pt.which ? b->seq2 : b->seq1) + (lo + pt.pair) * HP;
                            uint8_t* ql = (pt.which ? b->qual2 : b->qual1) + (lo + pt.pair) * HP;
                            sq[pt.pos] = pt.base; ql[pt.pos] = pt.qual;
                        }
                    };
                    const uint32_t nt = np >= 65536 ? 4u : 1u;
                    std::thread extra[3];
                    for (uint32_t t = 1; t < nt; t++) extra[t - 1] = std::thread(apply_range, (uint32_t)((uint64_t)np * t / nt), (uint32_t)((uint64_t)np * (t + 1) / nt));
                    apply_range(0, (uint32_t)((uint64_t)np / nt));
                    for (uint32_t t = 1; t < nt; t++) extra[t - 1].join();
                }
                if (hp_n)                                        /* caller's list: pair index relative to the whole host batch */
                    for (uint32_t i = 0; i < np; i++) {
                        if (*hp_n < hp_cap) { hp_out[*hp_n] = P[i]; hp_out[*hp_n].pair = (uint32_t)(lo + P[i].pair); }
                        (*hp_n)++;
                    }
            } else if (pk) {
                /* packed input: the list is the only way corrections reach the caller, and the kernel did not list all of this chunk's */
                if (hp_n) return set_err(FP_E_TOOLARGE, "base corrections of one host chunk exceed its patch list: the packed entry point cannot return them "
                                                        "all (use fp_process_pe_host_patches, which writes the corrected rows back)");
            } else {   /* patch list overflow: take the corrected rows wholesale (row by row when the host pitch differs); the issuing loop
                          keeps the device slot until this is done (it sees the same count) */
                if (hp_n) *hp_n = ~(uint64_t)0 >> 1;             /* the caller's list cannot be complete */
                uint8_t* dst[4] = {b->seq1, b->qual1, b->seq2, b->qual2};
                for (int a4 = 0; a4 < 4; a4++)
                    CK(cudaMemcpy2D(dst[a4] + lo * HP, (size_t)HP, c->d_stage[slot][a4], (size_t)S, (size_t)HP, (size_t)pend[hs].cnt, cudaMemcpyDeviceToHost));
            }
        }
        pend[hs].active = false;
        return FP_OK;
    };
    /* FP_B_PACK2BIT: a team of host threads packs the bases of chunk k into pinned slot k % NS, up to two chunks ahead of the chunk whose
       copies are being issued; a slot is free again once finish() has seen the chunk that used it */
    struct Team {
        std::vector<std::thread> th;
        std::mutex mu;
        std::condition_variable cv_allowed, cv_done;           /* blocking waits: spinning threads would eat the CPU quota the packers need */
        int64_t allowed = -1;
        bool stop = false;
        std::atomic<int> bad{0};
        std::vector<int> done;                                 /* [chunk] threads that finished it (under mu) */
        std::vector<std::vector<fp_npos>> nl;                  /* [thread * NS + slot] */
        ~Team() { { std::lock_guard<std::mutex> lk(mu); stop = true; } cv_allowed.notify_all(); for (auto& t : th) t.join(); }
    } team;
    const int NT = packfly ? (c->host_threads > 0 ? c->host_threads : default_host_threads()) : 0;
    if (packfly) {
        team.done.assign((size_t)nchunks, 0);
        team.nl.resize((size_t)NT * NS);
        team.allowed = 1;
        for (int t = 0; t < NT; t++)
            team.th.emplace_back([&, t]() {
                const int sides = pe ? 2 : 1;
                for (int64_t k = 0; k < nchunks; k++) {
                    {
                        std::unique_lock<std::mutex> lk(team.mu);
                        team.cv_allowed.wait(lk, [&] { return team.stop || team.allowed >= k; });
                        if (team.stop) return;
                    }
                    const int64_t lo = k * CH, cnt = std::min(CH, n - lo);
                    const int64_t r0 = cnt * t / NT, r1 = cnt * (t + 1) / NT;
                    std::vector<fp_npos>& nl = team.nl[(size_t)t * NS + (size_t)(k % NS)];
                    nl.clear();
                    for (int64_t r = r0; r < r1; r++)
                        for (int sd = 0; sd < sides; sd++) {
                            const int L = (sd ? b->len2 : b->len1)[lo + r];
                            if (L > HP) { team.bad.store(2); break; }
                            if (fp_pack_bases_row((sd ? b->seq2 : b->seq1) + (lo + r) * HP, L, c->h_pkb[k % NS][sd] + r * PB, (uint32_t)r, sd, nl)) { team.bad.store(1); break; }
                        }
                    bool last;
                    { std::lock_guard<std::mutex> lk(team.mu); last = ++team.done[(size_t)k] == NT; }
                    if (last) team.cv_done.notify_all();
                }
            });
    }
    /* Completion work of a chunk (waiting for its stream, corrected bases written back into the caller's rows, event / patch lists) runs
       on a helper thread when there are enough chunks, so that it overlaps the issue of the following chunks instead of delaying them:
       with 0.7 corrections per pair the write-back alone is a couple of milliseconds per chunk. */
    struct Fin {
        std::thread th;
        std::mutex mu;
        std::condition_variable cv;
        int64_t issued = 0, finished = 0;
        bool stop = false;
        int rc = FP_OK;
        std::string err;
        ~Fin() { { std::lock_guard<std::mutex> lk(mu); stop = true; } cv.notify_all(); if (th.joinable()) th.join(); }
    } fin;
    const bool use_fin = nchunks > 2;
    if (use_fin)
        fin.th = std::thread([&]() {
            cudaSetDevice(c->device);
            for (int64_t k = 0; k < nchunks; k++) {
                {
                    std::unique_lock<std::mutex> lk(fin.mu);
                    fin.cv.wait(lk, [&] { return fin.stop || fin.issued > k; });
                    if (fin.issued <= k) return;
                }
                const int r = finish(k);
                {
                    std::lock_guard<std::mutex> lk(fin.mu);
                    if (r && !fin.rc) { fin.rc = r; fin.err = g_err; }
                    fin.finished = k + 1;
                }
                fin.cv.notify_all();
            }
        });
    auto fin_wait = [&](int64_t need) -> int {                 /* until `need` chunks are finished (or the helper failed) */
        std::unique_lock<std::mutex> lk(fin.mu);
        fin.cv.wait(lk, [&] { return fin.finished >= need || fin.rc; });
        if (fin.rc) return set_err(fin.rc, "%s", fin.err.c_str());
        return FP_OK;
    };
    const bool trace = getenv("FP_TRACE_HOST") != nullptr;
    auto now = [] { return std::chrono::steady_clock::now(); };
    auto ms_since = [&](std::chrono::steady_clock::time_point t0) { return std::chrono::duration<double, std::milli>(now() - t0).count(); };
    double t_slot = 0, t_fin = 0, t_pack = 0, t_issue = 0;
    const auto t_begin = now();
    for (int64_t ci = 0; ci < nchunks; ci++) {
        const int slot = (int)(ci & 1);
        auto tp = now();
        if (!use_fin) rc = ci >= 2 ? finish(ci - 2) : FP_OK;    /* the slot's previous chunk is through */
        else if (ci >= 2) {
            /* the device slot is free once chunk ci - 2 has left the GPU; its host-side work may still be running on the helper -- unless
               that work needs the device buffers (adapter events, a patch list that overflowed): then wait for it.  The host buffers
               rotate over four chunks. */
            const int64_t k2 = ci - 2;
            CK(cudaEventSynchronize(c->chunk_done[k2 & 3]));
            t_slot += ms_since(tp); tp = now();
            const bool needs_dev = want_ev || (pe && c->p.correction_enabled && *c->h_npatch[k2 & 3] > c->patch_cap);
            rc = fin_wait(needs_dev ? ci - 1 : std::max<int64_t>(ci - 3, 0));
            t_fin += ms_since(tp); tp = now();
        }
        if (rc) return rc;
        if (packfly) {
            { std::lock_guard<std::mutex> lk(team.mu); team.allowed = ci + 2; }
            team.cv_allowed.notify_all();
            { std::unique_lock<std::mutex> lk(team.mu); team.cv_done.wait(lk, [&] { return team.done[(size_t)ci] >= NT; }); }
            t_pack += ms_since(tp); tp = now();
            if (team.bad.load() == 1) return set_err(FP_E_UNSUPPORTED, "a base outside {A,C,G,T,N}: not representable in packed rows (FP_B_PACK2BIT)");
            if (team.bad.load() == 2) return set_err(FP_E_INVAL, "a read is longer than the host row pitch");
        }
        const int64_t lo = ci * CH, cnt = std::min(CH, n - lo);
        cudaStream_t st = c->stream[slot];
        const size_t bytes = (size_t)cnt * S;
        if (pk) {
            /* packed rows up, then a small kernel restores the stride rows in HBM (6 TB/s: nothing next to the PCIe transfer) */
            const size_t bb = (size_t)cnt * pk->pitch_b, qb = (size_t)cnt * pk->pitch_q;
            CK(cudaMemcpyAsync(c->d_pk[slot][0], pk->bases1 + lo * pk->pitch_b, bb, cudaMemcpyHostToDevice, st));
            CK(cudaMemcpyAsync(c->d_pk[slot][1], pk->qual1 + lo * pk->pitch_q, qb, cudaMemcpyHostToDevice, st));
            CK(cudaMemcpyAsync(c->d_stage_len[slot][0], pk->len1 + lo, (size_t)cnt * 2, cudaMemcpyHostToDevice, st));
            if (pe) {
                CK(cudaMemcpyAsync(c->d_pk[slot][2], pk->bases2 + lo * pk->pitch_b, bb, cudaMemcpyHostToDevice, st));
                CK(cudaMemcpyAsync(c->d_pk[slot][3], pk->qual2 + lo * pk->pitch_q, qb, cudaMemcpyHostToDevice, st));
                CK(cudaMemcpyAsync(c->d_stage_len[slot][1], pk->len2 + lo, (size_t)cnt * 2, cudaMemcpyHostToDevice, st));
                CK(cudaMemsetAsync(c->d_npatch[slot], 0, 4, st));
            }
            const long long thr = (long long)cnt * (S >> 4);
            fp_unpack_kernel<<<(unsigned)((thr + 255) / 256), 256, 0, st>>>(c->d_pk[slot][0], c->d_pk[slot][1], c->d_stage_len[slot][0], cnt, pk->pitch_b, pk->pitch_q, S,
                                                                          c->d_stage[slot][0], c->d_stage[slot][1]);
            if (pe) fp_unpack_kernel<<<(unsigned)((thr + 255) / 256), 256, 0, st>>>(c->d_pk[slot][2], c->d_pk[slot][3], c->d_stage_len[slot][1], cnt, pk->pitch_b, pk->pitch_q, S,
                                                                                  c->d_stage[slot][2], c->d_stage[slot][3]);
            /* the chunk's slice of the sorted 'N' list */
            const fp_npos* nb0 = std::lower_bound(pk->npos, pk->npos + pk->n_npos, (uint32_t)lo, [](const fp_npos& e, uint32_t v) { return e.unit < v; });
            const fp_npos* nb1 = std::lower_bound(nb0, (const fp_npos*)(pk->npos + pk->n_npos), (uint32_t)(lo + cnt), [](const fp_npos& e, uint32_t v) { return e.unit < v; });
            const long long nn = nb1 - nb0;
            if (nn > 0) {
                if ((size_t)nn > c->npos_cap) {
                    CK(cudaDeviceSynchronize());
                    for (int i = 0; i < 2; i++) { cudaFree(c->d_npos[i]); CK(cudaMalloc(&c->d_npos[i], (size_t)(nn + nn / 2 + 1024) * sizeof(fp_npos))); }
                    c->npos_cap = (size_t)(nn + nn / 2 + 1024);
                }
                CK(cudaMemcpyAsync(c->d_npos[slot], nb0, (size_t)nn * sizeof(fp_npos), cudaMemcpyHostToDevice, st));
                fp_unpack_n_kernel<<<(unsigned)((nn + 255) / 256), 256, 0, st>>>(c->d_npos[slot], nn, lo, S, c->d_stage[slot][0], pe ? c->d_stage[slot][2] : nullptr);
            }
            CK(cudaGetLastError());
        } else if (packfly) {
            const int hs = (int)(ci % NS);
            size_t nn = 0;
            for (int t = 0; t < NT; t++) nn += team.nl[(size_t)t * NS + hs].size();
            if (nn > c->h_np_cap) {                                /* the slots' older chunks are done (finish above): safe to re-allocate */
                CK(cudaDeviceSynchronize());
                const size_t cap = nn + nn / 2 + 4096;
                for (int i = 0; i < NS; i++) { if (c->h_np[i]) cudaFreeHost(c->h_np[i]); c->h_np[i] = nullptr; CK(cudaMallocHost(&c->h_np[i], cap * sizeof(fp_npos))); }
                c->h_np_cap = cap;
            }
            if (nn > c->npos_cap) {
                CK(cudaDeviceSynchronize());
                for (int i = 0; i < 2; i++) { cudaFree(c->d_npos[i]); c->d_npos[i] = nullptr; CK(cudaMalloc(&c->d_npos[i], (nn + nn / 2 + 1024) * sizeof(fp_npos))); }
                c->npos_cap = nn + nn / 2 + 1024;
            }
            size_t o = 0;
            for (int t = 0; t < NT; t++) { const auto& v = team.nl[(size_t)t * NS + hs]; if (!v.empty()) memcpy(c->h_np[hs] + o, v.data(), v.size() * sizeof(fp_npos)); o += v.size(); }
            const size_t bb = (size_t)cnt * PB, qb = (size_t)cnt * HP;
            CK(cudaMemcpyAsync(c->d_pk[slot][0], c->h_pkb[hs][0], bb, cudaMemcpyHostToDevice, st));
            CK(cudaMemcpyAsync(c->d_pk[slot][1], b->qual1 + lo * HP, qb, cudaMemcpyHostToDevice, st));
            CK(cudaMemcpyAsync(c->d_stage_len[slot][0], b->len1 + lo, (size_t)cnt * 2, cudaMemcpyHostToDevice, st));
            if (pe) {
                CK(cudaMemcpyAsync(c->d_pk[slot][2], c->h_pkb[hs][1], bb, cudaMemcpyHostToDevice, st));
                CK(cudaMemcpyAsync(c->d_pk[slot][3], b->qual2 + lo * HP, qb, cudaMemcpyHostToDevice, st));
                CK(cudaMemcpyAsync(c->d_stage_len[slot][1], b->len2 + lo, (size_t)cnt * 2, cudaMemcpyHostToDevice, st));
                CK(cudaMemsetAsync(c->d_npatch[slot], 0, 4, st));
            }
            const long long thr = (long long)cnt * (S >> 4);
            fp_unpack_kernel<<<(unsigned)((thr + 255) / 256), 256, 0, st>>>(c->d_pk[slot][0], c->d_pk[slot][1], c->d_stage_len[slot][0], cnt, PB, HP, S, c->d_stage[slot][0], c->d_stage[slot][1]);
            if (pe) fp_unpack_kernel<<<(unsigned)((thr + 255) / 256), 256, 0, st>>>(c->d_pk[slot][2], c->d_pk[slot][3], c->d_stage_len[slot][1], cnt, PB, HP, S, c->d_stage[slot][2], c->d_stage[slot][3]);
            if (nn > 0) {
                CK(cudaMemcpyAsync(c->d_npos[slot], c->h_np[hs], nn * sizeof(fp_npos), cudaMemcpyHostToDevice, st));
                fp_unpack_n_kernel<<<(unsigned)((nn + 255) / 256), 256, 0, st>>>(c->d_npos[slot], (long long)nn, 0, S, c->d_stage[slot][0], pe ? c->d_stage[slot][2] : nullptr);
            }
            CK(cudaGetLastError());
        } else if (repitch) {
            const size_t hb = (size_t)cnt * HP;
            const uint8_t* src[4] = {b->seq1, b->qual1, b->seq2, b->qual2};
            CK(cudaMemcpyAsync(c->d_stage_len[slot][0], b->len1 + lo, (size_t)cnt * 2, cudaMemcpyHostToDevice, st));
            if (pe) { CK(cudaMemcpyAsync(c->d_stage_len[slot][1], b->len2 + lo, (size_t)cnt * 2, cudaMemcpyHostToDevice, st)); CK(cudaMemsetAsync(c->d_npatch[slot], 0, 4, st)); }
            const long long thr = (long long)cnt * (S >> 4);
            for (int k = 0; k < (pe ? 4 : 2); k++) {
                CK(cudaMemcpyAsync(c->d_pk[slot][k], src[k] + lo * HP, hb, cudaMemcpyHostToDevice, st));
                fp_repitch_kernel<<<(unsigned)((thr + 255) / 256), 256, 0, st>>>(c->d_pk[slot][k], c->d_stage_len[slot][k >> 1], cnt, HP, S, c->d_stage[slot][k]);
            }
            CK(cudaGetLastError());
        } else {
        CK(cudaMemcpyAsync(c->d_stage[slot][0], b->seq1 + lo * S, bytes, cudaMemcpyHostToDevice, st));
        CK(cudaMemcpyAsync(c->d_stage[slot][1], b->qual1 + lo * S, bytes, cudaMemcpyHostToDevice, st));
        CK(cudaMemcpyAsync(c->d_stage_len[slot][0], b->len1 + lo, (size_t)cnt * 2, cudaMemcpyHostToDevice, st));
        if (pe) {
            CK(cudaMemcpyAsync(c->d_stage[slot][2], b->seq2 + lo * S, bytes, cudaMemcpyHostToDevice, st));
            CK(cudaMemcpyAsync(c->d_stage[slot][3], b->qual2 + lo * S, bytes, cudaMemcpyHostToDevice, st));
            CK(cudaMemcpyAsync(c->d_stage_len[slot][1], b->len2 + lo, (size_t)cnt * 2, cudaMemcpyHostToDevice, st));
            CK(cudaMemsetAsync(c->d_npatch[slot], 0, 4, st));
        }
        }
        if (want_ev) {
            CK(cudaMemsetAsync(c->d_nev[slot], 0, 4, st));
            c->ev_dev = c->d_ev[slot]; c->ev_cap = c->ev_chunk_cap; c->ev_count = c->d_nev[slot];
        }
        fp_batch db;
        memset(&db, 0, sizeof(db));
        db.n = cnt; db.stride = S;
        if (b->flags & FP_B_INDEXED) { db.flags = FP_B_INDEXED; db.first_read_index = b->first_read_index + lo; }
        db.seq1 = c->d_stage[slot][0]; db.qual1 = c->d_stage[slot][1]; db.len1 = c->d_stage_len[slot][0];
        if (pe) { db.seq2 = c->d_stage[slot][2]; db.qual2 = c->d_stage[slot][3]; db.len2 = c->d_stage_len[slot][1]; }
        /* the over-representation sampling state (running counts, rank scratch) is one per ctx: chunk k+1's kernels wait for chunk
           k's (its H2D copies, issued above, still overlap them) */
        if (c->p.overrep_enabled) {
            if (!c->ovr_ev) CK(cudaEventCreateWithFlags(&c->ovr_ev, cudaEventDisableTiming));
            else CK(cudaStreamWaitEvent(st, c->ovr_ev, 0));
        }
        rc = launch_chain(c, &db, c->d_out[slot][0], pe ? c->d_out[slot][1] : nullptr, pe ? c->d_ov[slot] : nullptr,
                          pe ? c->d_patch[slot] : nullptr, c->patch_cap, pe ? c->d_npatch[slot] : nullptr, st);
        if (rc) return rc;
        if (c->p.overrep_enabled) CK(cudaEventRecord(c->ovr_ev, st));
        if (want_ev) CK(cudaMemcpyAsync(c->h_nev[slot], c->d_nev[slot], 4, cudaMemcpyDeviceToHost, st));
        CK(cudaMemcpyAsync(out1 + lo, c->d_out[slot][0], (size_t)cnt * sizeof(fp_read_result), cudaMemcpyDeviceToHost, st));
        if (pe) {
            CK(cudaMemcpyAsync(out2 + lo, c->d_out[slot][1], (size_t)cnt * sizeof(fp_read_result), cudaMemcpyDeviceToHost, st));
            if (ov) CK(cudaMemcpyAsync(ov + lo, c->d_ov[slot], (size_t)cnt * sizeof(fp_ov_result), cudaMemcpyDeviceToHost, st));
            if (c->p.correction_enabled) {
                CK(cudaMemcpyAsync(c->h_npatch[ci & 3], c->d_npatch[slot], 4, cudaMemcpyDeviceToHost, st));
                CK(cudaMemcpyAsync(c->h_patch[ci & 3], c->d_patch[slot], (size_t)c->patch_cap * sizeof(fp_patch), cudaMemcpyDeviceToHost, st));
            }
        }
        CK(cudaEventRecord(c->chunk_done[ci & 3], st));
        pend[ci & 3].lo = lo; pend[ci & 3].cnt = cnt; pend[ci & 3].active = true;
        if (use_fin) { { std::lock_guard<std::mutex> lk(fin.mu); fin.issued = ci + 1; } fin.cv.notify_all(); }
        t_issue += ms_since(tp);
    }
    const double t_loop = ms_since(t_begin);
    if (use_fin) { rc = fin_wait(nchunks); if (rc) return rc; }
    else for (int64_t k = std::max<int64_t>(nchunks - 2, 0); k < nchunks; k++) { rc = finish(k); if (rc) return rc; }
    if (trace)
        fprintf(stderr, "[fastp_b200 host] %lld units, %lld chunks, mode %s: issue loop %.2f ms (waiting: device slot %.2f, helper %.2f, packers %.2f; issuing %.2f), drain %.2f ms\n",
                (long long)n, (long long)nchunks, pk ? "packed" : packfly ? "pack2bit" : repitch ? "tight" : "rows", t_loop, t_slot, t_fin, t_pack, t_issue, ms_since(t_begin) - t_loop);
    return FP_OK;
}

extern "C" int fp_process_se_host(fp_ctx* c, const fp_batch* b, fp_read_result* out1) {
    if (!c || !b || !out1) return set_err(FP_E_INVAL, "null argument");
    if (c->p.paired) return set_err(FP_E_INVAL, "ctx was created for paired-end data");
    return process_host(c, b, out1, nullptr, nullptr);
}

extern "C" int fp_process_pe_host(fp_ctx* c, const fp_batch* b, fp_read_result* out1, fp_read_result* out2, fp_ov_result* ov) {
    if (!c || !b || !out1 || !out2) return set_err(FP_E_INVAL, "null argument");
    if (!c->p.paired) return set_err(FP_E_INVAL, "ctx was created for single-end data");
    return process_host(c, b, out1, out2, ov);
}

extern "C" int fp_process_se_host_packed(fp_ctx* c, const fp_packed_batch* pb, fp_read_result* out1) {
    if (!c || !pb || !out1) return set_err(FP_E_INVAL, "null argument");
    if (c->p.paired) return set_err(FP_E_INVAL, "ctx was created for paired-end data");
    fp_batch b; memset(&b, 0, sizeof(b));
    b.n = pb->n; b.stride = c->stride; b.flags = pb->flags; b.first_read_index = pb->first_read_index;
    return process_host(c, &b, out1, nullptr, nullptr, nullptr, 0, nullptr, pb);
}

extern "C" int fp_process_pe_host_packed(fp_ctx* c, const fp_packed_batch* pb, fp_read_result* out1, fp_read_result* out2, fp_ov_result* ov,
                                         fp_patch* patches, uint64_t patch_cap, uint64_t* n_patches) {
    if (!c || !pb || !out1 || !out2 || (patch_cap > 0 && (!patches || !n_patches))) return set_err(FP_E_INVAL, "null argument");
    if (!c->p.paired) return set_err(FP_E_INVAL, "ctx was created for single-end data");
    fp_batch b; memset(&b, 0, sizeof(b));
    b.n = pb->n; b.stride = c->stride; b.flags = pb->flags; b.first_read_index = pb->first_read_index;
    return process_host(c, &b, out1, out2, ov, patches, patch_cap, n_patches, pb);
}

extern "C" int fp_process_pe_host_patches(fp_ctx* c, const fp_batch* b, fp_read_result* out1, fp_read_result* out2, fp_ov_result* ov,
                                          fp_patch* patches, uint64_t patch_cap, uint64_t* n_patches) {
    if (!c || !b || !out1 || !out2 || !n_patches || (patch_cap > 0 && !patches)) return set_err(FP_E_INVAL, "null argument");
    if (!c->p.paired) return set_err(FP_E_INVAL, "ctx was created for single-end data");
    return process_host(c, b, out1, out2, ov, patches, patch_cap, n_patches);
}

/* ---------------- FASTQ text <-> rows (fp_fastq.cuh) ---------------- */
static int fq_ensure(fp_ctx::Buf& b, size_t need) {
    if (need <= b.cap) return FP_OK;
    if (b.p) cudaFree(b.p);
    b.p = nullptr; b.cap = 0;
    size_t cap = need + need / 4 + 256;
    CK(cudaMalloc(&b.p, cap));
    b.cap = cap;
    return FP_OK;
}

static_assert(sizeof(fp_fastq_rec) == sizeof(fq_rec), "fp_fastq_rec layout");

/* rec_end_out (optional, host): consumed bytes if only the first k records are kept is read later through fq_recend.
   il: interleaved text, mate 1 rows in d_seq .. d_recs and mate 2 rows in il's side 1; capacity and info->n_records count pairs. */
static int fastq_decode_impl(fp_ctx* c, const uint8_t* d_text, int64_t nbytes, int32_t final_chunk, int32_t phred64,
                             uint8_t* d_seq, uint8_t* d_qual, uint16_t* d_len, int64_t capacity, fp_fastq_rec* d_recs,
                             fp_fastq_info* info, fp_ctx::Buf& recend, const fq_side_rows* il = nullptr) {
    if (!c || !info || (nbytes > 0 && !d_text)) return set_err(FP_E_INVAL, "null argument");
    if (nbytes < 0 || nbytes >= ((int64_t)1 << 32) - 16) return set_err(FP_E_TOOLARGE, "FASTQ chunk must be smaller than 4 GiB");
    if (capacity < 0 || (capacity > 0 && (!d_seq || !d_qual || !d_len || !d_recs))) return set_err(FP_E_INVAL, "null row buffers");
    if (il && capacity > 0 && (!il->seq[1] || !il->qual[1] || !il->len[1] || !il->recs[1])) return set_err(FP_E_INVAL, "null row buffers");
    memset(info, 0, sizeof(*info));
    info->error_record = -1;
    if (nbytes == 0) return FP_OK;
    CK(cudaSetDevice(c->device));
    cudaStream_t st = c->stream[0];
    const int nbb = (int)((nbytes + FQ_BB - 1) / FQ_BB);
    int rc;
    if ((rc = fq_ensure(c->fq_bcnt, (size_t)(nbb + 1) * 4))) return rc;
    if ((rc = fq_ensure(c->fq_info, 64))) return rc;
    /* control words come back through MAPPED pinned host memory written by the kernels themselves: a small cudaMemcpy would queue
       behind the bulk text transfers on the copy engines (milliseconds when the text path is streaming) */
    if (!c->fq_hinfo) { CK(cudaHostAlloc((void**)&c->fq_hinfo, 256, cudaHostAllocMapped)); CK(cudaHostGetDevicePointer((void**)&c->fq_hinfo_dev, c->fq_hinfo, 0)); }
    volatile unsigned int* h_info = c->fq_hinfo;
    unsigned int* m_info = c->fq_hinfo_dev;
    unsigned int* d_info = (unsigned int*)c->fq_info.p;
    fq_term_count_kernel<<<nbb, FQ_T, 0, st>>>(d_text, nbytes, (unsigned int*)c->fq_bcnt.p);
    fq_term_scan_kernel<<<1, 32, 0, st>>>((unsigned int*)c->fq_bcnt.p, nbb, d_text, nbytes, final_chunk, nullptr, 0, m_info);
    CK(cudaStreamSynchronize(st));
    const unsigned int nlines = h_info[0], nterm = h_info[1];
    info->n_lines = nlines;
    if (nlines == 0) return FP_OK;
    if ((rc = fq_ensure(c->fq_term, (size_t)(nlines + 2) * 4))) return rc;
    unsigned int* d_term = (unsigned int*)c->fq_term.p;
    fq_term_fill_kernel<<<nbb, FQ_T, 0, st>>>(d_text, nbytes, (unsigned int*)c->fq_bcnt.p, d_term, nlines + 1);
    if (nlines > nterm) fq_set_u32_kernel<<<1, 1, 0, st>>>(d_term + nterm, (unsigned int)nbytes);     /* virtual terminator after the last byte */
    /* record automaton over the lines */
    const int nlb = (int)((nlines + FQ_LB - 1) / FQ_LB);
    if ((rc = fq_ensure(c->fq_agg, (size_t)nlb * sizeof(fq_elem)))) return rc;
    if ((rc = fq_ensure(c->fq_bstate, (size_t)nlb * 4))) return rc;
    if ((rc = fq_ensure(c->fq_brec, (size_t)nlb * 4))) return rc;
    fq_fsm_kernel<0><<<nlb, FQ_T, 0, st>>>(d_text, nbytes, d_term, nlines, (fq_elem*)c->fq_agg.p, nullptr, nullptr, nullptr, 0);
    fq_fsm_scan_kernel<<<1, 32, 0, st>>>((const fq_elem*)c->fq_agg.p, nlb, (unsigned int*)c->fq_bstate.p, (unsigned int*)c->fq_brec.p, m_info);
    CK(cudaStreamSynchronize(st));
    const unsigned int nstarted = h_info[2], ncomplete = h_info[3];
    if ((rc = fq_ensure(c->fq_recline, (size_t)(nstarted + 1) * 4))) return rc;
    unsigned int* d_recline = (unsigned int*)c->fq_recline.p;
    if (nstarted > 0)
        fq_fsm_kernel<1><<<nlb, FQ_T, 0, st>>>(d_text, nbytes, d_term, nlines, nullptr, (const unsigned int*)c->fq_bstate.p, (const unsigned int*)c->fq_brec.p,
                                               d_recline, nstarted);
    const unsigned int nrec = (unsigned int)std::min<int64_t>(ncomplete, il ? 2 * capacity : capacity);
    fq_side_rows S{};
    if (il) { S = *il; S.seq[0] = d_seq; S.qual[0] = d_qual; S.len[0] = d_len; S.recs[0] = reinterpret_cast<fq_rec*>(d_recs); }
    if (nrec > 0) {
        if ((rc = fq_ensure(recend, (size_t)nrec * 4))) return rc;
        CK(cudaMemsetAsync(d_info + 8, 0xFF, 4, st));             /* first bad record = none */
        if (il)
            fq_scatter_il_kernel<<<(nrec + FQ_T / 32 - 1) / (FQ_T / 32), FQ_T, 0, st>>>(d_text, nbytes, d_term, d_recline, nrec, c->stride, phred64, S,
                                                                                          (unsigned int*)recend.p, d_info + 8, d_info + 9);
        else
            fq_scatter_kernel<<<(nrec + FQ_T / 32 - 1) / (FQ_T / 32), FQ_T, 0, st>>>(d_text, nbytes, d_term, d_recline, nrec, c->stride, phred64,
                                                                                       d_seq, d_qual, d_len, reinterpret_cast<fq_rec*>(d_recs),
                                                                                       (unsigned int*)recend.p, d_info + 8, d_info + 9);
    }
    if (il)
        fq_finish_il_kernel<<<1, 1, 0, st>>>(d_term, nlines, nterm, nbytes, final_chunk, d_recline, nstarted, ncomplete, nrec, S.recs[0], S.recs[1],
                                             d_info + 8, m_info + 8);
    else
        fq_finish_kernel<<<1, 1, 0, st>>>(d_term, nlines, nterm, nbytes, d_recline, nstarted, ncomplete, nrec, reinterpret_cast<const fq_rec*>(d_recs), d_info + 8, m_info + 8);
    CK(cudaGetLastError());
    CK(cudaStreamSynchronize(st));
    info->n_records = h_info[8];
    info->error = (int32_t)h_info[9];
    info->error_record = h_info[10] == 0xFFFFFFFFu ? -1 : (int64_t)h_info[10];
    info->more = (int32_t)h_info[11];
    info->consumed = (int64_t)h_info[12] | ((int64_t)h_info[13] << 32);
    return FP_OK;
}

extern "C" int fp_fastq_decode(fp_ctx* c, const uint8_t* d_text, int64_t nbytes, int32_t final_chunk, int32_t phred64,
                               uint8_t* d_seq, uint8_t* d_qual, uint16_t* d_len, int64_t capacity, fp_fastq_rec* d_recs,
                               fp_fastq_info* info) {
    if (!c) return set_err(FP_E_INVAL, "null argument");
    return fastq_decode_impl(c, d_text, nbytes, final_chunk, phred64, d_seq, d_qual, d_len, capacity, d_recs, info, c->fq_recend);
}

extern "C" int fp_fastq_decode_interleaved(fp_ctx* c, const uint8_t* d_text, int64_t nbytes, int32_t final_chunk, int32_t phred64,
                                           uint8_t* d_seq1, uint8_t* d_qual1, uint16_t* d_len1, fp_fastq_rec* d_recs1,
                                           uint8_t* d_seq2, uint8_t* d_qual2, uint16_t* d_len2, fp_fastq_rec* d_recs2,
                                           int64_t capacity, fp_fastq_info* info) {
    if (!c) return set_err(FP_E_INVAL, "null argument");
    if (capacity >= ((int64_t)1 << 30)) return set_err(FP_E_TOOLARGE, "capacity must be below 2^30 pairs");
    fq_side_rows il{};
    il.seq[1] = d_seq2; il.qual[1] = d_qual2; il.len[1] = d_len2; il.recs[1] = reinterpret_cast<fq_rec*>(d_recs2);
    return fastq_decode_impl(c, d_text, nbytes, final_chunk, phred64, d_seq1, d_qual1, d_len1, capacity, d_recs1, info, c->fq_recend, &il);
}

/* size pass, scan and write pass of one output stream (fp_fastq.cuh); M is unused by FQ_SEL_PLAIN */
template <int SEL>
static int fastq_encode_impl(fp_ctx* c, const uint8_t* d_text, const fp_fastq_rec* d_recs, const fp_read_result* d_res,
                             const uint8_t* d_seq, const uint8_t* d_qual, const fq_merge_args& M, int64_t n, uint8_t* d_out, int64_t out_cap, int64_t* out_bytes) {
    CK(cudaSetDevice(c->device));
    cudaStream_t st = c->stream[0];
    const int nblk = (int)((n + FQ_SCAN_ITEMS - 1) / FQ_SCAN_ITEMS);
    int rc;
    if ((rc = fq_ensure(c->fq_bsum, (size_t)(nblk + 1) * 8))) return rc;
    unsigned long long* d_bs = (unsigned long long*)c->fq_bsum.p;
    fq_size_blocksum_kernel<SEL><<<nblk, FQ_T, 0, st>>>(d_text, reinterpret_cast<const fq_rec*>(d_recs), d_res, M, n, d_bs);
    if (!c->fq_hinfo) { CK(cudaHostAlloc((void**)&c->fq_hinfo, 256, cudaHostAllocMapped)); CK(cudaHostGetDevicePointer((void**)&c->fq_hinfo_dev, c->fq_hinfo, 0)); }
    fq_size_scan_kernel<<<1, 32, 0, st>>>(d_bs, nblk, reinterpret_cast<unsigned long long*>(c->fq_hinfo_dev + 32));
    fq_encode_kernel<SEL><<<nblk, FQ_T, 0, st>>>(d_text, reinterpret_cast<const fq_rec*>(d_recs), d_res, d_seq, d_qual, M, c->stride, n, d_bs, d_out,
                                                 (unsigned long long)std::max<int64_t>(out_cap, 0));
    CK(cudaGetLastError());
    CK(cudaStreamSynchronize(st));
    *out_bytes = (int64_t)*reinterpret_cast<volatile unsigned long long*>(c->fq_hinfo + 32);
    return FP_OK;
}

extern "C" int fp_fastq_encode(fp_ctx* c, const uint8_t* d_text, const fp_fastq_rec* d_recs, const fp_read_result* d_res,
                               const uint8_t* d_seq, const uint8_t* d_qual, int64_t n, uint8_t* d_out, int64_t out_cap, int64_t* out_bytes) {
    if (!c || !out_bytes) return set_err(FP_E_INVAL, "null argument");
    *out_bytes = 0;
    if (n <= 0) return FP_OK;
    if (!d_text || !d_recs || !d_res || !d_seq || !d_qual || (out_cap > 0 && !d_out)) return set_err(FP_E_INVAL, "null argument");
    return fastq_encode_impl<FQ_SEL_PLAIN>(c, d_text, d_recs, d_res, d_seq, d_qual, fq_merge_args{}, n, d_out, out_cap, out_bytes);
}

extern "C" int fp_fastq_encode_interleaved(fp_ctx* c, const uint8_t* d_text1, const fp_fastq_rec* d_recs1, const uint8_t* d_text2, const fp_fastq_rec* d_recs2,
                                           const fp_read_result* d_res1, const fp_read_result* d_res2,
                                           const uint8_t* d_seq1, const uint8_t* d_qual1, const uint8_t* d_seq2, const uint8_t* d_qual2,
                                           int64_t n, uint8_t* d_out, int64_t out_cap, int64_t* out_bytes) {
    if (!c || !out_bytes) return set_err(FP_E_INVAL, "null argument");
    *out_bytes = 0;
    if (!c->p.paired) return set_err(FP_E_INVAL, "ctx was created for single-end data: interleaved output needs pairs");
    if (c->p.merge_enabled) return set_err(FP_E_INVAL, "ctx merges pairs: its stdout stream is the merged one (fp_fastq_encode_merge)");
    if (n <= 0) return FP_OK;
    if (!d_text1 || !d_recs1 || !d_text2 || !d_recs2 || !d_res1 || !d_res2 || !d_seq1 || !d_qual1 || !d_seq2 || !d_qual2 || (out_cap > 0 && !d_out))
        return set_err(FP_E_INVAL, "null argument");
    fq_merge_args M{};
    M.text2 = d_text2; M.recs2 = reinterpret_cast<const fq_rec*>(d_recs2); M.res2 = d_res2; M.seq2 = d_seq2; M.qual2 = d_qual2;
    return fastq_encode_impl<FQ_SEL_INTERLEAVED>(c, d_text1, d_recs1, d_res1, d_seq1, d_qual1, M, n, d_out, out_cap, out_bytes);
}

extern "C" int fp_fastq_encode_merge(fp_ctx* c, int32_t which, const uint8_t* d_text1, const fp_fastq_rec* d_recs1, const uint8_t* d_text2, const fp_fastq_rec* d_recs2,
                                     const fp_read_result* d_res1, const fp_read_result* d_res2, const fp_ov_result* d_ov,
                                     const uint8_t* d_seq1, const uint8_t* d_qual1, const uint8_t* d_seq2, const uint8_t* d_qual2,
                                     int64_t n, uint8_t* d_out, int64_t out_cap, int64_t* out_bytes) {
    if (!c || !out_bytes) return set_err(FP_E_INVAL, "null argument");
    *out_bytes = 0;
    if (!c->p.paired) return set_err(FP_E_INVAL, "ctx was created for single-end data: merging needs pairs");
    if (!c->p.merge_enabled) return set_err(FP_E_INVAL, "ctx was created without merge_enabled (fp_fastq_encode writes its output)");
    if (which != FP_FQ_OUT_MERGED && which != FP_FQ_OUT_R1 && which != FP_FQ_OUT_R2) return set_err(FP_E_INVAL, "which must be FP_FQ_OUT_MERGED, FP_FQ_OUT_R1 or FP_FQ_OUT_R2");
    if (n <= 0) return FP_OK;
    if (!d_text1 || !d_recs1 || !d_text2 || !d_recs2 || !d_res1 || !d_res2 || !d_ov || !d_seq1 || !d_qual1 || !d_seq2 || !d_qual2 || (out_cap > 0 && !d_out))
        return set_err(FP_E_INVAL, "null argument");
    fq_merge_args M{};
    M.ov = d_ov; M.include_unmerged = c->p.merge_include_unmerged ? 1 : 0;
    if (which == FP_FQ_OUT_R2) {                                  /* side 2 is written, side 1 only gives its records */
        M.res2 = d_res1;
        return fastq_encode_impl<FQ_SEL_SIDE>(c, d_text2, d_recs2, d_res2, d_seq2, d_qual2, M, n, d_out, out_cap, out_bytes);
    }
    M.text2 = d_text2; M.recs2 = reinterpret_cast<const fq_rec*>(d_recs2); M.res2 = d_res2; M.seq2 = d_seq2; M.qual2 = d_qual2;
    if (which == FP_FQ_OUT_R1) return fastq_encode_impl<FQ_SEL_SIDE>(c, d_text1, d_recs1, d_res1, d_seq1, d_qual1, M, n, d_out, out_cap, out_bytes);
    return fastq_encode_impl<FQ_SEL_MERGED>(c, d_text1, d_recs1, d_res1, d_seq1, d_qual1, M, n, d_out, out_cap, out_bytes);
}

/* the argument rules of fp_fastq_encode_rejects and fp_fastq_process_host_outs (options.cpp:136-143, :222-229) */
static int fastq_rejects_check(const fp_ctx* c, int writers) {
    if (writers & ~(FP_FQ_W_UNPAIRED1 | FP_FQ_W_UNPAIRED2)) return set_err(FP_E_INVAL, "writers holds bits other than FP_FQ_W_UNPAIRED1 / FP_FQ_W_UNPAIRED2");
    if (writers && !c->p.paired) return set_err(FP_E_INVAL, "unpaired outputs need a paired ctx (the reference ignores them for single-end data)");
    if (writers && c->p.merge_enabled && c->p.merge_include_unmerged)
        return set_err(FP_E_INVAL, "unpaired outputs with merge_include_unmerged (the reference ignores them: every pair is merged or written whole)");
    return FP_OK;
}

extern "C" int fp_fastq_encode_rejects(fp_ctx* c, int32_t which, int32_t writers, const uint8_t* d_text1, const fp_fastq_rec* d_recs1,
                                       const uint8_t* d_text2, const fp_fastq_rec* d_recs2, const fp_read_result* d_res1, const fp_read_result* d_res2,
                                       const uint8_t* d_seq1, const uint8_t* d_qual1, const uint16_t* d_len1,
                                       const uint8_t* d_seq2, const uint8_t* d_qual2, const uint16_t* d_len2,
                                       int64_t n, uint8_t* d_out, int64_t out_cap, int64_t* out_bytes) {
    if (!c || !out_bytes) return set_err(FP_E_INVAL, "null argument");
    *out_bytes = 0;
    if (which != FP_FQ_OUT_UNPAIRED1 && which != FP_FQ_OUT_UNPAIRED2 && which != FP_FQ_OUT_FAILED)
        return set_err(FP_E_INVAL, "which must be FP_FQ_OUT_UNPAIRED1, FP_FQ_OUT_UNPAIRED2 or FP_FQ_OUT_FAILED");
    if (which != FP_FQ_OUT_FAILED && !c->p.paired) return set_err(FP_E_INVAL, "unpaired outputs need a paired ctx (the reference ignores them for single-end data)");
    int rc;
    if ((rc = fastq_rejects_check(c, writers))) return rc;
    if (n <= 0) return FP_OK;
    const bool pe = c->p.paired != 0;
    if (!d_text1 || !d_recs1 || !d_res1 || !d_seq1 || !d_qual1 || !d_len1 || (out_cap > 0 && !d_out) ||
        (pe && (!d_text2 || !d_recs2 || !d_res2 || !d_seq2 || !d_qual2 || !d_len2)))
        return set_err(FP_E_INVAL, "null argument");
    fq_merge_args M{};
    M.len1 = d_len1; M.writers = writers; M.merging = pe && c->p.merge_enabled; M.include_unmerged = c->p.merge_include_unmerged ? 1 : 0;
    if (pe) { M.text2 = d_text2; M.recs2 = reinterpret_cast<const fq_rec*>(d_recs2); M.res2 = d_res2; M.seq2 = d_seq2; M.qual2 = d_qual2; M.len2 = d_len2; }
    if (which == FP_FQ_OUT_UNPAIRED1) return fastq_encode_impl<FQ_SEL_UNPAIRED1>(c, d_text1, d_recs1, d_res1, d_seq1, d_qual1, M, n, d_out, out_cap, out_bytes);
    if (which == FP_FQ_OUT_UNPAIRED2) return fastq_encode_impl<FQ_SEL_UNPAIRED2>(c, d_text1, d_recs1, d_res1, d_seq1, d_qual1, M, n, d_out, out_cap, out_bytes);
    return fastq_encode_impl<FQ_SEL_FAILED>(c, d_text1, d_recs1, d_res1, d_seq1, d_qual1, M, n, d_out, out_cap, out_bytes);
}

/* The round loop of the text path.  outs / ocap / out_bytes are indexed by FP_FQ_OUT_*; a NULL buffer is not encoded.  merging: the ctx
   merges pairs, so every round also keeps the chain's overlap results for the merged stream.  The reject streams read the round's decoded
   lengths (fqh_len, which the chain leaves as they are) and take the unpaired writers from which unpaired buffers are given. */
static int fastq_process_host_impl(fp_ctx* c, const uint8_t* text1, int64_t nbytes1, const uint8_t* text2, int64_t nbytes2,
                                   int32_t final_chunk, int32_t phred64, uint8_t* const outs[FP_FQ_OUTS], const int64_t ocap[FP_FQ_OUTS],
                                   int64_t* const out_bytes[FP_FQ_OUTS],
                                   int64_t* n_units, int64_t* consumed1, int64_t* consumed2, fp_fastq_info* info1, fp_fastq_info* info2) {
    const int sides = c->p.paired ? 2 : 1;
    const bool merging = c->p.merge_enabled && sides == 2;
    const int writers = (outs[FP_FQ_OUT_UNPAIRED1] ? FP_FQ_W_UNPAIRED1 : 0) | (outs[FP_FQ_OUT_UNPAIRED2] ? FP_FQ_W_UNPAIRED2 : 0);
    /* fp_fastq_set_interleaved: mates alternate in text1 (one upload, one decode per round); out1 receives read 1 and read 2 of every pair */
    const bool il_in = c->fq_il_in && sides == 2, il_out = c->fq_il_out && sides == 2 && !merging;
    if (c->dup_flags) return set_err(FP_E_INVAL, "duplicate flags are set (fp_set_dup_flags): the text path runs its own duplicate filter (fp_fastq_set_dedup)");
    if (il_in && (text2 || nbytes2 != 0)) return set_err(FP_E_INVAL, "interleaved input: both mates are in text1 (pass text2 NULL and nbytes2 0)");
    if (il_out && outs[FP_FQ_OUT_R2]) return set_err(FP_E_INVAL, "interleaved output: both reads go to out1 (pass no out2 buffer)");
    CK(cudaSetDevice(c->device));
    cudaStream_t st = c->stream[0], up = c->stream[1];
    if (!c->fq_stream_out) {
        CK(cudaStreamCreateWithFlags(&c->fq_stream_out, cudaStreamNonBlocking));
        CK(cudaEventCreateWithFlags(&c->fq_ev_up, cudaEventDisableTiming));
        for (int k = 0; k < 2; k++) CK(cudaEventCreateWithFlags(&c->fq_ev_out[k], cudaEventDisableTiming));
    }
    cudaStream_t outst = c->fq_stream_out;
    const uint8_t* text[2] = {text1, text2};
    const int64_t nb[2] = {nbytes1, sides == 2 && !il_in ? nbytes2 : 0};
    const int64_t cap = c->max_batch;
    /* The text goes up in pieces on its own stream while the pieces already on the device are decoded, run through the chain and
       encoded, and the previous round's output text goes down on a third stream: H2D, kernels and D2H overlap inside ONE call
       (pinned host buffers assumed; pageable ones still work, serialised).  A piece is a fraction of a device batch of text; the
       host never has to find record borders -- the decode of a prefix reports what it consumed and the next round starts there. */
    const int64_t piece = std::max<int64_t>((int64_t)4 << 20, std::min<int64_t>((int64_t)64 << 20, cap * (int64_t)(2 * c->stride + 64) / 4));
    int rc;
    for (int s = 0; s < sides; s++) {
        if ((rc = fq_ensure(c->fqh_text[s], (size_t)nb[s] + 64))) return rc;
        if ((rc = fq_ensure(c->fqh_seq[s], (size_t)cap * c->stride + 64))) return rc;
        if ((rc = fq_ensure(c->fqh_qual[s], (size_t)cap * c->stride + 64))) return rc;
        if ((rc = fq_ensure(c->fqh_len[s], (size_t)cap * 2))) return rc;
        if ((rc = fq_ensure(c->fqh_recs[s], (size_t)cap * sizeof(fp_fastq_rec)))) return rc;
        if ((rc = fq_ensure(c->fqh_res[s], (size_t)cap * sizeof(fp_read_result)))) return rc;
    }
    if (merging && (rc = fq_ensure(c->fqh_ov, (size_t)cap * sizeof(fp_ov_result)))) return rc;
    int64_t upl[2] = {0, 0}, start[2] = {0, 0}, obytes[FP_FQ_OUTS] = {0}, units = 0;
    fp_fastq_info agg[2]; memset(agg, 0, sizeof(agg)); agg[0].error_record = agg[1].error_record = -1;
    int flip = 0;
    auto upload_more = [&]() -> int {
        bool any = false;
        for (int s = 0; s < sides; s++) {
            const int64_t n = std::min(piece, nb[s] - upl[s]);
            if (n > 0) { CK(cudaMemcpyAsync((uint8_t*)c->fqh_text[s].p + upl[s], text[s] + upl[s], (size_t)n, cudaMemcpyHostToDevice, up)); upl[s] += n; any = true; }
        }
        if (any) CK(cudaEventRecord(c->fq_ev_up, up));
        return FP_OK;
    };
    if ((rc = upload_more())) return rc;
    const bool trace = getenv("FP_FQ_TRACE") != nullptr;
    auto now = []() { timespec t; clock_gettime(CLOCK_MONOTONIC, &t); return t.tv_sec * 1e3 + t.tv_nsec * 1e-6; };
    const double t_begin = now();
    for (;;) {
        const double t0 = now();
        CK(cudaStreamWaitEvent(st, c->fq_ev_up, 0));             /* this round reads what has been issued so far ... */
        const int64_t have[2] = {upl[0], upl[1]}, rstart[2] = {start[0], start[1]};
        const bool saw_all = have[0] >= nb[0] && have[1] >= nb[1];
        if ((rc = upload_more())) return rc;                      /* ... while the next piece flies */
        fp_fastq_info inf[2]; memset(inf, 0, sizeof(inf));
        int fin[2];
        fq_side_rows il{};
        il.seq[1] = (uint8_t*)c->fqh_seq[1].p; il.qual[1] = (uint8_t*)c->fqh_qual[1].p; il.len[1] = (uint16_t*)c->fqh_len[1].p;
        il.recs[1] = (fq_rec*)c->fqh_recs[1].p;
        const int decodes = il_in ? 1 : sides;
        for (int s = 0; s < decodes; s++) {
            fin[s] = (final_chunk && have[s] >= nb[s]) ? 1 : 0;
            rc = fastq_decode_impl(c, (const uint8_t*)c->fqh_text[s].p + rstart[s], have[s] - rstart[s], fin[s], phred64, (uint8_t*)c->fqh_seq[s].p,
                                   (uint8_t*)c->fqh_qual[s].p, (uint16_t*)c->fqh_len[s].p, cap, (fp_fastq_rec*)c->fqh_recs[s].p, &inf[s], c->fqh_recend[s],
                                   il_in ? &il : nullptr);
            if (rc) return rc;
        }
        const double t1 = now();
        int64_t n = inf[0].n_records;
        if (sides == 2 && !il_in) n = std::min(n, inf[1].n_records);   /* pairs end with the shorter input (FastqReaderPair::read) */
        bool reader_ended = false;                                /* a reader hit a record it rejects: it returns NULL, the stream ends */
        for (int s = 0; s < decodes; s++) {
            int64_t used = inf[s].consumed;
            if (n != inf[s].n_records) {                          /* this side decoded more records than the pair count: keep only n */
                used = 0;                                         /* resume right after record n-1 (end offsets were kept per side) */
                if (n > 0) {
                    fq_copy_u32_kernel<<<1, 1, 0, st>>>((const unsigned int*)c->fqh_recend[s].p + (n - 1), c->fq_hinfo_dev + 48);
                    CK(cudaStreamSynchronize(st));
                    used = *reinterpret_cast<volatile unsigned int*>(c->fq_hinfo + 48);
                }
            } else if (inf[s].error != FP_FQ_OK) {
                reader_ended = true;
                agg[s].error = inf[s].error; agg[s].error_record = agg[s].n_records + inf[s].error_record;
            }
            agg[s].n_records += n; agg[s].n_lines += inf[s].n_lines;
            start[s] = rstart[s] + used;
        }
        if (n > 0) {
            fp_batch b; memset(&b, 0, sizeof(b));
            b.n = n; b.stride = c->stride;
            b.seq1 = (uint8_t*)c->fqh_seq[0].p; b.qual1 = (uint8_t*)c->fqh_qual[0].p; b.len1 = (uint16_t*)c->fqh_len[0].p;
            if (sides == 2) { b.seq2 = (uint8_t*)c->fqh_seq[1].p; b.qual2 = (uint8_t*)c->fqh_qual[1].p; b.len2 = (uint16_t*)c->fqh_len[1].p; }
            const uint8_t* saved_flags = c->dup_flags;
            if (c->fq_dup_level > 0) {                            /* Duplicate::checkRead / checkPair on the reads as read, before the chain (:397-401) */
                if ((rc = fq_ensure(c->fq_dupflags, (size_t)cap))) return rc;
                if ((rc = fp_dup_check(c, &b, c->fq_dup_level, (uint8_t*)c->fq_dupflags.p, st))) return rc;
                if (c->fq_dedup) c->dup_flags = (const uint8_t*)c->fq_dupflags.p;
            }
            struct FlagsBack { fp_ctx* c; const uint8_t* f; ~FlagsBack() { c->dup_flags = f; } } flags_back{c, saved_flags};
            if (sides == 2) {
                rc = launch_chain(c, &b, (fp_read_result*)c->fqh_res[0].p, (fp_read_result*)c->fqh_res[1].p, merging ? (fp_ov_result*)c->fqh_ov.p : nullptr,
                                  nullptr, 0, nullptr, st);
            } else rc = launch_chain(c, &b, (fp_read_result*)c->fqh_res[0].p, nullptr, nullptr, nullptr, 0, nullptr, st);
            if (rc) return rc;
            CK(cudaEventSynchronize(c->fq_ev_out[flip]));        /* the output buffers of two rounds ago have gone down */
            const uint8_t* rtext[2] = {(const uint8_t*)c->fqh_text[0].p + rstart[0], sides == 2 ? (const uint8_t*)c->fqh_text[1].p + rstart[1] : nullptr};
            if (il_in) rtext[1] = rtext[0];                       /* both mates' records point into the one text */
            for (int s = 0; s < FP_FQ_OUTS; s++) {
                if (!outs[s]) continue;                           /* caller does not want this stream's text */
                fp_ctx::Buf& ob = c->fqh_outbuf[flip][s];
                const int64_t room = std::max<int64_t>(ocap[s] - obytes[s], 0);
                /* per unit: one record of a side; on the merged stream one read of up to two rows, or two records; on the failed stream two
                   tagged records */
                const bool two = s == FP_FQ_OUT_MERGED || s == FP_FQ_OUT_FAILED || (il_out && s == FP_FQ_OUT_R1);
                int64_t want = std::min<int64_t>(room, n * (int64_t)(two ? 4 * c->stride + 512 : 2 * c->stride + 256));
                int64_t total = 0;
                const fp_fastq_rec* recs[2] = {(const fp_fastq_rec*)c->fqh_recs[0].p, (const fp_fastq_rec*)c->fqh_recs[1].p};
                const fp_read_result* res[2] = {(const fp_read_result*)c->fqh_res[0].p, (const fp_read_result*)c->fqh_res[1].p};
                const uint8_t* seq[2] = {(const uint8_t*)c->fqh_seq[0].p, (const uint8_t*)c->fqh_seq[1].p};
                const uint8_t* qual[2] = {(const uint8_t*)c->fqh_qual[0].p, (const uint8_t*)c->fqh_qual[1].p};
                for (int attempt = 0; attempt < 2; attempt++) {   /* names longer than the estimate: encode again into a buffer of the exact size */
                    if ((rc = fq_ensure(ob, (size_t)want + 64))) return rc;
                    if (s >= FP_FQ_OUT_UNPAIRED1)
                        rc = fp_fastq_encode_rejects(c, s, writers, rtext[0], recs[0], rtext[1], recs[1], res[0], res[1], seq[0], qual[0],
                                                     (const uint16_t*)c->fqh_len[0].p, seq[1], qual[1], (const uint16_t*)c->fqh_len[1].p,
                                                     n, (uint8_t*)ob.p, want, &total);
                    else if (il_out)                              /* s == FP_FQ_OUT_R1: an out2 buffer was refused above */
                        rc = fp_fastq_encode_interleaved(c, rtext[0], recs[0], rtext[1], recs[1], res[0], res[1], seq[0], qual[0], seq[1], qual[1],
                                                         n, (uint8_t*)ob.p, want, &total);
                    else if (merging)
                        rc = fp_fastq_encode_merge(c, s, rtext[0], recs[0], rtext[1], recs[1], res[0], res[1], (const fp_ov_result*)c->fqh_ov.p,
                                                   seq[0], qual[0], seq[1], qual[1], n, (uint8_t*)ob.p, want, &total);
                    else {
                        const int side = s == FP_FQ_OUT_R2 ? 1 : 0;
                        rc = fp_fastq_encode(c, rtext[side], recs[side], res[side], seq[side], qual[side], n, (uint8_t*)ob.p, want, &total);
                    }
                    if (rc) return rc;
                    if (total <= want) break;
                    if (total > room) return set_err(FP_E_TOOLARGE, "output buffer too small for the encoded FASTQ text");
                    want = total;
                }
                if (total > 0) CK(cudaMemcpyAsync(outs[s] + obytes[s], ob.p, (size_t)total, cudaMemcpyDeviceToHost, outst));
                obytes[s] += total;
            }
            CK(cudaEventRecord(c->fq_ev_out[flip], outst));
            flip ^= 1;
            units += n;
        }
        if (trace) fprintf(stderr, "[fq] round t=%.2f ms: decode %.2f, rest %.2f, n=%lld have=%lld/%lld\n", t0 - t_begin, t1 - t0, now() - t1, (long long)n, (long long)have[0], (long long)nb[0]);
        if (reader_ended) break;
        if (n == 0 && saw_all) break;                             /* nothing more can become complete in this call */
    }
    const double t_loop = now();
    CK(cudaStreamSynchronize(up));
    CK(cudaStreamSynchronize(st));
    CK(cudaStreamSynchronize(outst));
    if (trace) fprintf(stderr, "[fq] loop %.2f ms, drain %.2f ms\n", t_loop - t_begin, now() - t_loop);
    agg[0].consumed = start[0]; agg[1].consumed = start[1];
    if (il_in) memset(&agg[1], 0, sizeof(agg[1]));
    *n_units = units; *consumed1 = start[0]; if (consumed2) *consumed2 = start[1];
    for (int s = 0; s < FP_FQ_OUTS; s++) if (out_bytes[s]) *out_bytes[s] = obytes[s];
    if (info1) *info1 = agg[0];
    if (info2 && sides == 2) *info2 = agg[1];
    return FP_OK;
}

extern "C" int fp_fastq_process_host(fp_ctx* c, const uint8_t* text1, int64_t nbytes1, const uint8_t* text2, int64_t nbytes2,
                                     int32_t final_chunk, int32_t phred64,
                                     uint8_t* out1, int64_t out_cap1, int64_t* out_bytes1,
                                     uint8_t* out2, int64_t out_cap2, int64_t* out_bytes2,
                                     int64_t* n_units, int64_t* consumed1, int64_t* consumed2, fp_fastq_info* info1, fp_fastq_info* info2) {
    if (!c || !n_units || !consumed1 || !out_bytes1) return set_err(FP_E_INVAL, "null argument");
    if (c->p.paired && (!consumed2 || !out_bytes2)) return set_err(FP_E_INVAL, "paired ctx needs the second side");
    if (c->p.paired && c->p.merge_enabled) return set_err(FP_E_INVAL, "ctx merges pairs: use fp_fastq_process_host_merge, which also returns the merged reads");
    uint8_t* const outs[FP_FQ_OUTS] = {nullptr, out1, c->p.paired ? out2 : nullptr, nullptr, nullptr, nullptr};
    const int64_t ocap[FP_FQ_OUTS] = {0, out_cap1, out_cap2, 0, 0, 0};
    int64_t* const ob[FP_FQ_OUTS] = {nullptr, out_bytes1, out_bytes2, nullptr, nullptr, nullptr};
    return fastq_process_host_impl(c, text1, nbytes1, text2, nbytes2, final_chunk, phred64, outs, ocap, ob, n_units, consumed1, consumed2, info1, info2);
}

extern "C" int fp_fastq_process_host_merge(fp_ctx* c, const uint8_t* text1, int64_t nbytes1, const uint8_t* text2, int64_t nbytes2,
                                           int32_t final_chunk, int32_t phred64,
                                           uint8_t* out1, int64_t out_cap1, int64_t* out_bytes1,
                                           uint8_t* out2, int64_t out_cap2, int64_t* out_bytes2,
                                           uint8_t* merged, int64_t merged_cap, int64_t* merged_bytes,
                                           int64_t* n_units, int64_t* consumed1, int64_t* consumed2, fp_fastq_info* info1, fp_fastq_info* info2) {
    if (!c || !n_units || !consumed1 || !consumed2 || !out_bytes1 || !out_bytes2 || !merged_bytes) return set_err(FP_E_INVAL, "null argument");
    if (!c->p.paired) return set_err(FP_E_INVAL, "ctx was created for single-end data: merging needs pairs");
    if (!c->p.merge_enabled) return set_err(FP_E_INVAL, "ctx was created without merge_enabled: use fp_fastq_process_host");
    uint8_t* const outs[FP_FQ_OUTS] = {merged, out1, out2, nullptr, nullptr, nullptr};
    const int64_t ocap[FP_FQ_OUTS] = {merged_cap, out_cap1, out_cap2, 0, 0, 0};
    int64_t* const ob[FP_FQ_OUTS] = {merged_bytes, out_bytes1, out_bytes2, nullptr, nullptr, nullptr};
    return fastq_process_host_impl(c, text1, nbytes1, text2, nbytes2, final_chunk, phred64, outs, ocap, ob, n_units, consumed1, consumed2, info1, info2);
}

extern "C" int fp_fastq_process_host_outs(fp_ctx* c, const uint8_t* text1, int64_t nbytes1, const uint8_t* text2, int64_t nbytes2,
                                          int32_t final_chunk, int32_t phred64, uint8_t* const outs[FP_FQ_OUTS], const int64_t out_caps[FP_FQ_OUTS],
                                          int64_t out_bytes[FP_FQ_OUTS], int64_t* n_units, int64_t* consumed1, int64_t* consumed2,
                                          fp_fastq_info* info1, fp_fastq_info* info2) {
    if (!c || !outs || !out_caps || !out_bytes || !n_units || !consumed1) return set_err(FP_E_INVAL, "null argument");
    if (c->p.paired && !consumed2) return set_err(FP_E_INVAL, "paired ctx needs the second side");
    if (!c->p.paired && outs[FP_FQ_OUT_R2]) return set_err(FP_E_INVAL, "an out2 buffer on a single-end ctx");
    if (outs[FP_FQ_OUT_MERGED] && !(c->p.paired && c->p.merge_enabled)) return set_err(FP_E_INVAL, "a merged buffer on a ctx that does not merge pairs");
    const int writers = (outs[FP_FQ_OUT_UNPAIRED1] ? FP_FQ_W_UNPAIRED1 : 0) | (outs[FP_FQ_OUT_UNPAIRED2] ? FP_FQ_W_UNPAIRED2 : 0);
    int rc;
    if ((rc = fastq_rejects_check(c, writers))) return rc;
    int64_t* ob[FP_FQ_OUTS];
    for (int s = 0; s < FP_FQ_OUTS; s++) ob[s] = &out_bytes[s];
    return fastq_process_host_impl(c, text1, nbytes1, text2, nbytes2, final_chunk, phred64, outs, out_caps, ob, n_units, consumed1, consumed2, info1, info2);
}

/* ---------------- duplication bloom filter (fp_dup.h / fp_dup.cuh) ---------------- */
extern "C" int fp_dup_check(fp_ctx* c, const fp_batch* b, int32_t accuracy_level, uint8_t* d_is_dup, void* stream) {
    if (!c || !b) return set_err(FP_E_INVAL, "null argument");
    if (b->n < 0 || b->n >= ((int64_t)1 << 31)) return set_err(FP_E_TOOLARGE, "batch larger than 2^31 (split it)");
    if (accuracy_level < 1 || accuracy_level > 6) return set_err(FP_E_INVAL, "dup accuracy level must be 1..6");
    CK(cudaSetDevice(c->device));
    cudaStream_t st = stream ? (cudaStream_t)stream : c->stream[0];
    const int paired = c->p.paired ? 1 : 0;
    if (!c->dup.bits) {                                        /* Duplicate::Duplicate src/duplicate.cpp:9-66 */
        uint64_t buf_bytes; int buf_num;
        fp_dup_sizes(accuracy_level, &buf_bytes, &buf_num);
        std::vector<uint64_t> primes((size_t)buf_num * FP_DUP_PRIME_LEN);
        fp_dup_primes(primes.data(), (int)primes.size());
        /* built in locals and committed only when every step has succeeded (a 32 GiB level-6 allocation can fail) */
        uint32_t* bits = nullptr; uint64_t* d_primes = nullptr; unsigned long long* d_count = nullptr;
        cudaError_t e1 = cudaMalloc(&bits, (size_t)buf_num * buf_bytes);
        if (e1 == cudaSuccess) e1 = cudaMemset(bits, 0, (size_t)buf_num * buf_bytes);
        if (e1 == cudaSuccess) e1 = cudaMalloc(&d_primes, primes.size() * 8);
        if (e1 == cudaSuccess) e1 = cudaMemcpy(d_primes, primes.data(), primes.size() * 8, cudaMemcpyHostToDevice);
        if (e1 == cudaSuccess) e1 = cudaMalloc(&d_count, 8);
        if (e1 == cudaSuccess) e1 = cudaMemset(d_count, 0, 8);
        if (e1 != cudaSuccess) { cudaFree(bits); cudaFree(d_primes); cudaFree(d_count); return set_err(FP_E_CUDA, "duplicate filter state: %s", cudaGetErrorString(e1)); }
        c->dup.bits = bits; c->d_dup_primes = d_primes; c->d_dup_count = d_count;
        c->dup.buf_num = buf_num; c->dup.buf_bits = buf_bytes << 3; c->dup.offset_mask = (uint64_t)FP_DUP_PRIME_LEN * buf_num - 1;
        c->dup.primes = c->d_dup_primes;
        c->dup_level = accuracy_level; c->dup_total = 0;
    } else if (accuracy_level != c->dup_level) return set_err(FP_E_INVAL, "dup accuracy level differs from the first call's");
    const int64_t n = b->n;
    if (n == 0) return FP_OK;
    if (b->stride != c->stride) return set_err(FP_E_INVAL, "batch stride differs from the ctx stride");
    const int64_t total = n * c->dup.buf_num;
    uint64_t cap = 1; while (cap < (uint64_t)(2 * total + 16)) cap <<= 1;
    int rc;
    if ((rc = fq_ensure(c->dup_pos, (size_t)total * 8))) return rc;
    if ((rc = fq_ensure(c->dup_keys, (size_t)cap * 8))) return rc;
    if ((rc = fq_ensure(c->dup_vals, (size_t)cap * 4))) return rc;
    fp_dup_state S = c->dup;
    S.pos = (uint64_t*)c->dup_pos.p; S.keys = (uint64_t*)c->dup_keys.p; S.vals = (uint32_t*)c->dup_vals.p; S.table_mask = cap - 1;
    CK(cudaMemsetAsync(S.keys, 0xFF, (size_t)cap * 8, st));    /* FP_DUP_EMPTY */
    CK(cudaMemsetAsync(S.vals, 0xFF, (size_t)cap * 4, st));
    const unsigned gu = (unsigned)((n + 255) / 256), gt = (unsigned)((total + 255) / 256);
    fp_dup_hash_warp_kernel<<<(unsigned)((n + 7) / 8), 256, 0, st>>>(S, n, b->seq1, b->len1, b->seq2, b->len2, b->stride, paired);
    fp_dup_first_kernel<<<gt, 256, 0, st>>>(S, total);
    fp_dup_decide_kernel<<<gu, 256, 0, st>>>(S, n, d_is_dup, c->d_dup_count);
    fp_dup_commit_kernel<<<gt, 256, 0, st>>>(S, total);
    CK(cudaGetLastError());
    c->dup_total += n;
    return FP_OK;
}

extern "C" int fp_set_dup_flags(fp_ctx* c, const uint8_t* d_is_dup) {
    if (!c) return set_err(FP_E_INVAL, "null argument");
    c->dup_flags = d_is_dup;
    return FP_OK;
}

extern "C" int fp_fastq_set_dedup(fp_ctx* c, int32_t accuracy_level, int32_t dedup) {
    if (!c) return set_err(FP_E_INVAL, "null argument");
    if (accuracy_level < 0 || accuracy_level > 6) return set_err(FP_E_INVAL, "dup accuracy level must be 0 (off) .. 6");
    c->fq_dup_level = accuracy_level; c->fq_dedup = dedup ? 1 : 0;
    return FP_OK;
}

extern "C" int fp_fastq_set_interleaved(fp_ctx* c, int32_t in, int32_t out) {
    if (!c) return set_err(FP_E_INVAL, "null argument");
    if (in && !c->p.paired) return set_err(FP_E_INVAL, "interleaved input needs a paired ctx");
    if (out && !c->p.paired) return set_err(FP_E_INVAL, "interleaved output needs a paired ctx");
    if (out && c->p.merge_enabled) return set_err(FP_E_INVAL, "interleaved output on a ctx that merges pairs (its stdout stream is the merged one)");
    c->fq_il_in = in ? 1 : 0; c->fq_il_out = out ? 1 : 0;
    return FP_OK;
}

extern "C" int fp_dup_totals(fp_ctx* c, int64_t* total, int64_t* dups) {
    if (!c || !total || !dups) return set_err(FP_E_INVAL, "null argument");
    *total = c->dup_total; *dups = 0;
    if (!c->d_dup_count) return FP_OK;
    CK(cudaSetDevice(c->device));
    CK(cudaDeviceSynchronize());
    unsigned long long v = 0;
    CK(cudaMemcpy(&v, c->d_dup_count, 8, cudaMemcpyDeviceToHost));
    *dups = (int64_t)v;
    return FP_OK;
}

extern "C" int fp_dup_reset(fp_ctx* c) {
    if (!c) return set_err(FP_E_INVAL, "null argument");
    if (!c->dup.bits) return FP_OK;
    CK(cudaSetDevice(c->device));
    CK(cudaDeviceSynchronize());
    CK(cudaMemset(c->dup.bits, 0, (size_t)c->dup.buf_num * (c->dup.buf_bits >> 3)));
    CK(cudaMemset(c->d_dup_count, 0, 8));
    c->dup_total = 0;
    return FP_OK;
}

/* ---------------- counters ---------------- */
extern "C" int fp_counters_reset(fp_ctx* c) {
    if (!c) return set_err(FP_E_INVAL, "null argument");
    CK(cudaSetDevice(c->device));
    CK(cudaDeviceSynchronize());
    CK(cudaMemset(c->d_raw, 0, c->L.total * 8));
    c->reads_seen = 0;
    if (c->d_ovr_base) CK(cudaMemset(c->d_ovr_base, 0, 16));
    return FP_OK;
}

static int finalize(fp_ctx* c, cudaStream_t st) {
    const int threads = 256;
    const int blocks = (int)((c->L.total + threads - 1) / threads);
    fp_finalize_kernel<<<blocks, threads, 0, st>>>(c->d_raw, c->d_fin, c->L);
    CK(cudaGetLastError());
    return FP_OK;
}

extern "C" int fp_counters_fetch(fp_ctx* c, int64_t* host_out) {
    if (!c || !host_out) return set_err(FP_E_INVAL, "null argument");
    CK(cudaSetDevice(c->device));
    CK(cudaDeviceSynchronize());
    int rc = finalize(c, c->stream[0]);
    if (rc) return rc;
    CK(cudaMemcpyAsync(host_out, c->d_fin, c->L.total * 8, cudaMemcpyDeviceToHost, c->stream[0]));
    CK(cudaStreamSynchronize(c->stream[0]));
    return FP_OK;
}

extern "C" int fp_counters_device_ptr(fp_ctx* c, int64_t** dev_ptr, int64_t* n_words) {
    if (!c || !dev_ptr) return set_err(FP_E_INVAL, "null argument");
    CK(cudaSetDevice(c->device));
    CK(cudaDeviceSynchronize());
    /* the RAW block is what gets summed across ranks (totals are derived afterwards by fetch) */
    *dev_ptr = reinterpret_cast<int64_t*>(c->d_raw);
    if (n_words) *n_words = c->L.total;
    return FP_OK;
}

/* ncclAllReduce resolved at run time from the NCCL already in the process (torch bundles libnccl.so.2) */
typedef int (*nccl_allreduce_fn)(const void*, void*, size_t, int, int, void*, cudaStream_t);
extern "C" int fp_counters_allreduce(fp_ctx* c, void* comm, void* stream) {
    if (!c) return set_err(FP_E_INVAL, "null argument");
    if (!comm) return FP_OK;
    static nccl_allreduce_fn fn = nullptr;
    if (!fn) {
        void* h = dlopen("libnccl.so.2", RTLD_NOW | RTLD_NOLOAD);
        if (!h) h = dlopen("libnccl.so.2", RTLD_NOW);
        if (!h) h = dlopen("libnccl.so", RTLD_NOW);
        if (h) fn = (nccl_allreduce_fn)dlsym(h, "ncclAllReduce");
        if (!fn) return set_err(FP_E_UNSUPPORTED, "ncclAllReduce not found (libnccl.so.2 not loadable)");
    }
    CK(cudaSetDevice(c->device));
    cudaStream_t st = stream ? (cudaStream_t)stream : c->stream[0];
    /* stream-ordered: the caller enqueues it behind its fp_process_* calls on the same stream; fp_counters_fetch waits for the device */
    /* ncclInt64 = 4, ncclSum = 0 (nccl.h) */
    int rc = fn(c->d_raw, c->d_raw, (size_t)c->L.total, 4, 0, comm, st);
    if (rc != 0) return set_err(FP_E_CUDA, "ncclAllReduce failed");
    return FP_OK;
}

extern "C" int fp_host_alloc(void** p, size_t bytes) {
    if (!p) return set_err(FP_E_INVAL, "null argument");
    CK(cudaMallocHost(p, bytes));
    return FP_OK;
}
extern "C" int fp_host_free(void* p) {
    CK(cudaFreeHost(p));
    return FP_OK;
}

extern "C" int fp_synth_fill(fp_ctx* c, const fp_batch* b, int64_t first_index, uint64_t seed, int32_t profile, int32_t read_len, void* stream) {
    if (!c || !b) return set_err(FP_E_INVAL, "null argument");
    if (read_len > b->stride || read_len < 16) return set_err(FP_E_INVAL, "read_len must be in [16, stride]");
    CK(cudaSetDevice(c->device));
    cudaStream_t st = stream ? (cudaStream_t)stream : c->stream[0];
    if (b->n == 0) return FP_OK;
    const int threads = 128;
    const int blocks = (int)((b->n + threads - 1) / threads);
    fp_synth_kernel<<<blocks, threads, 0, st>>>(*b, first_index, seed, profile, read_len);
    CK(cudaGetLastError());
    return FP_OK;
}

extern "C" int fp_kernel_time_ms(fp_ctx* c, double* total_ms, int64_t* n_launches, int reset) {
    if (!c) return set_err(FP_E_INVAL, "null argument");
    CK(cudaSetDevice(c->device));
    int rc = drain_events(c);
    if (rc) return rc;
    if (total_ms) *total_ms = c->ev_ms;
    if (n_launches) *n_launches = c->ev_n;
    if (reset) { c->ev_ms = 0; c->ev_n = 0; }
    return FP_OK;
}

/* ---------------- host-side pre-scan: over-representation candidates ----------------
 * Evaluator::computeOverRepSeq (src/evaluator.cpp:78-169) over the first reads of one side, given as rows: count every
 * substring of length 10 / 20 / 40 / 100 / min(150, seqlen-2) of the reads until 151*10000 bases have been seen, keep those at
 * or above the per-length count thresholds, then drop a kept sequence that is a substring of another kept one unless it is at
 * least ten times as frequent (integer division, in the reference's map order).  Control plane, runs once per input on the
 * host like the reference's Evaluator; the result is what fp_params.overrep_seqs1/2 take.
 * The reference counts in a std::map<string,long> (about 5 M entries for 2x250 bp); here a first pass counts 64-bit substring
 * hashes in a flat table and only substrings whose HASH reaches the smallest threshold are counted exactly -- same set, same
 * counts (a colliding hash can only nominate a string whose exact count then fails the threshold). */
#include <map>
#include <unordered_map>
extern "C" int fp_host_overrep_candidates(const uint8_t* seq, const uint16_t* len, int64_t n, int32_t stride, int32_t seqlen,
                                          char* out, int64_t out_cap, int32_t* n_out, int64_t* bytes_out) {
    if (!seq || !len || !n_out || !bytes_out || n < 0 || stride <= 0) return set_err(FP_E_INVAL, "null argument");
    const long BASE_LIMIT = 151 * 10000;                                    /* evaluator.cpp:83 */
    const int steps[5] = {10, 20, 40, 100, std::min(150, seqlen - 2)};     /* :99 */
    auto threshold = [&](int L) -> long {                                   /* :116-140 */
        if (L >= seqlen - 1) return 3;
        if (L >= 100) return 5;
        if (L >= 40) return 20;
        if (L >= 20) return 100;
        if (L >= 10) return 500;
        return -1;
    };
    int64_t nreads = 0; long bases = 0;
    while (nreads < n && bases < BASE_LIMIT) { bases += len[nreads]; nreads++; }   /* :88-96: a read is taken whole once bases < limit */
    const unsigned long long B = 0x9E3779B97F4A7C15ull;
    std::unordered_map<unsigned long long, uint32_t> hcount;
    hcount.reserve((size_t)nreads * 1024);
    std::vector<unsigned long long> pref;
    for (int pass = 0; pass < 2; pass++) {
        std::map<std::string, long> exact;
        for (int64_t r = 0; r < nreads; r++) {
            const uint8_t* s = seq + (size_t)r * stride; const int rlen = len[r];
            pref.assign(rlen + 1, 0);
            for (int i = 0; i < rlen; i++) pref[i + 1] = pref[i] * B + (unsigned long long)(s[i] + 1);
            for (int k = 0; k < 5; k++) {
                const int step = steps[k];
                if (step <= 0) continue;
                unsigned long long bp = 1; for (int e = 0; e < step; e++) bp *= B;
                const long thr = threshold(step);
                for (int i = 0; i < rlen - step; i++) {                     /* :102 */
                    const unsigned long long h = (pref[i + step] - pref[i] * bp) ^ ((unsigned long long)step << 56);
                    if (pass == 0) hcount[h]++;
                    else if (thr >= 0 && (long)hcount[h] >= thr) exact[std::string((const char*)s + i, step)]++;
                }
            }
        }
        if (pass == 0) continue;
        std::map<std::string, long> hot;
        for (auto& kv : exact) { const long thr = threshold((int)kv.first.size()); if (thr >= 0 && kv.second >= thr) hot[kv.first] = kv.second; }
        for (auto it = hot.begin(); it != hot.end();) {                     /* :143-161 remove substrings, erasing while iterating */
            bool sub = false;
            for (auto it2 = hot.begin(); it2 != hot.end(); ++it2)
                if (it->first != it2->first && it2->first.find(it->first) != std::string::npos && it->second / it2->second < 10) { sub = true; break; }
            if (sub) it = hot.erase(it); else ++it;
        }
        int64_t used = 0; int32_t cnt = 0;
        for (auto& kv : hot) {
            const int64_t need = (int64_t)kv.first.size() + 1;
            if (out && used + need <= out_cap) memcpy(out + used, kv.first.c_str(), (size_t)need);
            used += need; cnt++;
        }
        *n_out = cnt; *bytes_out = used;
        if (used > out_cap) return set_err(FP_E_TOOLARGE, "candidate buffer too small (bytes_out holds the size needed)");
    }
    return FP_OK;
}
