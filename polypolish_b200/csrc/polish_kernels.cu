// polish_kernels.cu — host side of the polish hot path: context, device buffers, the launch sequence and the C-ABI entry
// points.  The kernels themselves (k_prep, k_bin_bounds, k_tile, k_compact, k_classify_multi) are in polish_dev.cuh, which
// also documents the design; DESIGN.md §3 has the derivation and the measurements.
#include <cuda_runtime.h>

#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>

#include <algorithm>
#include <functional>
#include <cstddef>
#include <cstdio>
#include <string>
#include <vector>

#include "pp_internal.h"
#include "pp_ctx.cuh"
#include "polish_dev.cuh"

// ------------------------------------------------------------------------------------------------------
// host side: context, buffers, entry points
// ------------------------------------------------------------------------------------------------------
// (DevBuf, the buffer ids and pp_ctx live in pp_ctx.cuh, shared with tok_kernels.cu)

static void init_comp_table(uint8_t* t) {
    for (int i = 0; i < 256; ++i) t[i] = 'N';
    const char* a = "ATGCNRYSWKMBVDH.-?";
    const char* b = "TACGNYRSWMKVBHD.-?";
    for (int i = 0; a[i]; ++i) t[(unsigned char)a[i]] = (uint8_t)b[i];
}

extern "C" const char* pp_version(void) { return "0.6.1-b200"; }

extern "C" void* pp_host_alloc(size_t bytes) {
    void* p = nullptr;
    if (cudaHostAlloc(&p, bytes ? bytes : 1, cudaHostAllocDefault) != cudaSuccess) { cudaGetLastError(); return nullptr; }
    return p;
}
extern "C" void pp_host_free(void* p) { if (p) cudaFreeHost(p); }

#define PP_INIT_IMAGE (64u << 10)     // the per-call reset block (statistics, status, options) travels as ONE small copy when it fits

extern "C" int pp_create(int device, pp_ctx** out) {
    if (!out) return PP_ERR_ARG;
    *out = nullptr;
    int n = 0;
    cudaError_t e = cudaGetDeviceCount(&n);
    if (e != cudaSuccess || n == 0 || device < 0 || device >= n) { cudaGetLastError(); return PP_ERR_CUDA; }   // no CPU fallback
    pp_ctx* ctx = new pp_ctx();
    ctx->device = device;
    if (cudaSetDevice(device) != cudaSuccess) { delete ctx; return PP_ERR_CUDA; }
    cudaDeviceProp prop;
    if (cudaGetDeviceProperties(&prop, device) != cudaSuccess || prop.major != 9 || prop.minor != 0) { delete ctx; return PP_ERR_CUDA; }   // sm_90a code loads on compute capability 9.0 only
    ctx->sm_count = prop.multiProcessorCount;
    if (cudaStreamCreateWithFlags(&ctx->stream, cudaStreamNonBlocking) != cudaSuccess) { delete ctx; return PP_ERR_CUDA; }
    if (cudaStreamCreateWithFlags(&ctx->copy_stream, cudaStreamNonBlocking) != cudaSuccess) { delete ctx; return PP_ERR_CUDA; }
    if (cudaEventCreateWithFlags(&ctx->ev_small, cudaEventDisableTiming) != cudaSuccess ||
        cudaEventCreateWithFlags(&ctx->ev_seq, cudaEventDisableTiming) != cudaSuccess) { delete ctx; return PP_ERR_CUDA; }
    for (auto& ev : ctx->ev) if (cudaEventCreate(&ev) != cudaSuccess) { delete ctx; return PP_ERR_CUDA; }
    if (cudaHostAlloc((void**)&ctx->h_status, sizeof(DevStatus), cudaHostAllocDefault) != cudaSuccess) { delete ctx; return PP_ERR_CUDA; }
    if (cudaHostAlloc((void**)&ctx->h_params, sizeof(DevParams), cudaHostAllocDefault) != cudaSuccess) { delete ctx; return PP_ERR_CUDA; }
    if (cudaHostAlloc((void**)&ctx->h_init, PP_INIT_IMAGE, cudaHostAllocDefault) != cudaSuccess) { delete ctx; return PP_ERR_CUDA; }
    uint8_t comp[256];
    init_comp_table(comp);
    if (cudaMemcpyToSymbol(c_comp, comp, 256) != cudaSuccess) { delete ctx; return PP_ERR_CUDA; }
    *out = ctx;
    return PP_OK;
}

extern "C" void pp_destroy(pp_ctx* ctx) {
    if (!ctx) return;
    cudaSetDevice(ctx->device);
    if (ctx->stream) cudaStreamSynchronize(ctx->stream);
    pp_tok_release(ctx);
    for (auto& b : ctx->b) b.release();
    for (auto& ev : ctx->ev) if (ev) cudaEventDestroy(ev);
    if (ctx->h_status) cudaFreeHost(ctx->h_status);
    if (ctx->h_params) cudaFreeHost(ctx->h_params);
    if (ctx->h_init) cudaFreeHost(ctx->h_init);
    if (ctx->ev_small) cudaEventDestroy(ctx->ev_small);
    if (ctx->ev_seq) cudaEventDestroy(ctx->ev_seq);
    if (ctx->copy_stream) cudaStreamDestroy(ctx->copy_stream);
    if (ctx->stream) cudaStreamDestroy(ctx->stream);
    delete ctx;
}

extern "C" const char* pp_last_error(const pp_ctx* ctx) { return ctx ? ctx->err.c_str() : "null context"; }

// internal (host_api.cpp, filter_kernels.cu): shared access to the context
int pp_ctx_fail(pp_ctx* ctx, int code, const char* msg) { ctx->err = msg; return code; }
int pp_ctx_device(pp_ctx* ctx) { return ctx->device; }
int pp_ctx_sm_count(pp_ctx* ctx) { return ctx->sm_count; }
cudaStream_t pp_ctx_stream(pp_ctx* ctx) { return ctx->stream; }
cudaEvent_t pp_ctx_event(pp_ctx* ctx, int i) { return ctx->ev[i]; }
void pp_ctx_count_launches(pp_ctx* ctx, uint32_t n) { ctx->launches = n; }
int pp_ctx_fail_cuda(pp_ctx* ctx, cudaError_t e, const char* what, const char* file, int line) {
    ctx->err = std::string("CUDA error: ") + cudaGetErrorString(e) + " at " + what + " (" + file + ":" + std::to_string(line) + ")";
    return PP_ERR_CUDA;
}
void* pp_ctx_scratch2(pp_ctx* ctx, size_t bytes) {
    if (ctx->b[B_SCRATCH2].ensure(bytes) != cudaSuccess) { cudaGetLastError(); return nullptr; }
    return ctx->b[B_SCRATCH2].p;
}
void* pp_ctx_scratch(pp_ctx* ctx, size_t bytes) {
    if (ctx->b[B_SCRATCH].ensure(bytes) != cudaSuccess) { cudaGetLastError(); return nullptr; }
    return ctx->b[B_SCRATCH].p;
}

template <class T>
static int upload(pp_ctx* ctx, int which, const T* src, size_t n, size_t pad_bytes = 64) {
    CK(ctx->b[which].ensure(n * sizeof(T) + pad_bytes));
    if (n) CK(cudaMemcpyAsync(ctx->b[which].p, src, n * sizeof(T), cudaMemcpyHostToDevice, ctx->stream));
    return PP_OK;
}

// Draft bases + contig offsets onto the device (shared by pp_dataset_upload and the SAM tokeniser).
int pp_ctx_upload_contigs(pp_ctx* ctx, const pp_contigs* c) {
    if (!c || !c->off || !c->bases || c->n_contigs == 0) return ctx->fail(PP_ERR_ARG, "null or empty contigs");
    const uint64_t G = c->off[c->n_contigs];
    if (G == 0 || G >= 0xFFFFFFFFull - 2 * VT_CHUNK) return ctx->fail(PP_ERR_ARG, "total assembly length must be in [1, 2^32-4096)");
    int rc;
    if ((rc = upload(ctx, B_DRAFT, c->bases, G, VT_CHUNK + 256))) return rc;
    if ((rc = upload(ctx, B_CTGOFF, c->off, (size_t)c->n_contigs + 1))) return rc;
    ctx->G = G; ctx->n_contigs = c->n_contigs;
    return PP_OK;
}

// The input side of DevData (alignment arrays, assembly, the binned dataset).
static void fill_data(pp_ctx* ctx, DevData& d) {
    const uint64_t G = ctx->G;
    memset(&d, 0, sizeof d);
    d.n_aln = ctx->n_aln;
    const DsArrays a = ds_view(ctx->b + B_CONTIG);
    d.contig = a.contig; d.ref_start = a.ref_start; d.read_id = a.read_id; d.seq_off = a.seq_off; d.cigar_off = a.cigar_off; d.nm = a.nm;
    d.cigar_ops = a.cigar_ops; d.seq_len = a.seq_len; d.n_cigar = a.n_cigar; d.flags = a.flags; d.seq_pool = a.seq_pool;
    d.draft = ctx->b[B_DRAFT].as<uint8_t>();
    d.contig_off = ctx->b[B_CTGOFF].as<unsigned long long>(); d.n_contigs = ctx->n_contigs; d.G = (uint32_t)G;
    d.n_bins = (uint32_t)((G + PP_BIN - 1) >> PP_BIN_SHIFT); d.n_tiles = (uint32_t)((G + TL_T - 1) / TL_T);
    d.recs = ctx->b[B_RECS].as<TileRec>(); d.key = ctx->b[B_KEY].as<uint32_t>(); d.val = ctx->b[B_VAL].as<uint32_t>();
    d.sval = ctx->b[B_SVAL].as<uint32_t>(); d.bin_start = ctx->b[B_BINSTART].as<uint32_t>();
    d.srec = ctx->b[B_SREC].as<TileRec>(); d.sseq = ctx->b[B_SSEQ].as<uint4>();
    d.n_slots = ctx->n_slots; d.max_ext = ctx->max_ext;
    d.tile_order = ctx->b[B_TILEORDER].as<uint32_t>();
    d.kf = ctx->b[B_KF].as<uint32_t>(); d.wrec = ctx->b[B_NK].as<uint4>(); d.errc = ctx->b[B_ERRC].as<uint8_t>(); d.gq = ctx->b[B_GQ].as<uint16_t>();
}

// Once per dataset (pp_dataset_upload, pp_tok_finish): the alignments binned by position.  k_bin (record + 256-position bin key of
// every alignment that can ever contribute) -> stable radix sort of (key, alignment) -> k_bin_bounds -> k_permute (records into
// slot order) -> k_permute_seq (the bases of the fast-path reads into slot order, forward strand).  Nothing here depends on the
// polish options: repeated pp_polish_resident calls reuse it, and pp_polish pays for it inside its own call.  Alignments that start
// at or past their contig's end wait for the bases: k_past_end trims them once seq_ready has run.
// `seq_ready`: run right before the first kernel that reads the sequence pool (pp_dataset_upload finishes the pool's upload there).
template <int BITS>
static int bin_dataset(pp_ctx* ctx, const std::function<int()>& seq_ready) {
    cudaStream_t s = ctx->stream;
    const uint64_t n_aln = ctx->n_aln, G = ctx->G;
    const uint32_t n_bins = (uint32_t)((G + PP_BIN - 1) >> PP_BIN_SHIFT);
    int key_bits = 1;
    while ((1ull << key_bits) < (uint64_t)n_bins + 2) key_bits++;
    const size_t na = (size_t)n_aln + 16;
    CK(ctx->b[B_RECS].ensure(na * sizeof(TileRec)));
    CK(ctx->b[B_KEY].ensure(na * 4)); CK(ctx->b[B_VAL].ensure(na * 4));
    CK(ctx->b[B_SKEY].ensure(na * 4)); CK(ctx->b[B_SVAL].ensure(na * 4));
    CK(ctx->b[B_BINSTART].ensure(((size_t)n_bins + 4) * 4));
    CK(ctx->b[B_ERRC].ensure(na)); CK(ctx->b[B_GQ].ensure(na * 2));
    CK(ctx->b[B_PARAMS].ensure(sizeof(DevParams) + 256 + sizeof(DevStatus)));
    size_t cub_bytes = 0;
    CK(cub::DeviceRadixSort::SortPairs(nullptr, cub_bytes, (const uint32_t*)nullptr, (uint32_t*)nullptr, (const uint32_t*)nullptr,
                                       (uint32_t*)nullptr, (int)n_aln, 0, key_bits, s));
    CK(ctx->b[B_CUBTMP].ensure(cub_bytes + 256));
    ctx->n_slots = 0; ctx->max_ext = 0;
    DevData d;
    fill_data(ctx, d);
    d.st = (DevStatus*)(ctx->b[B_PARAMS].as<uint8_t>() + 256);
    CK(cudaMemsetAsync(d.st, 0, sizeof(DevStatus), s));
    if (n_aln) {
        k_bin<BITS><<<(uint32_t)std::min<uint64_t>((n_aln + 255) / 256, (uint64_t)ctx->sm_count * 16), 256, 0, s>>>(d);
        CK(cub::DeviceRadixSort::SortPairs(ctx->b[B_CUBTMP].p, cub_bytes, d.key, ctx->b[B_SKEY].as<uint32_t>(), d.val,
                                           ctx->b[B_SVAL].as<uint32_t>(), (int)n_aln, 0, key_bits, s));   // stable: SAM order inside a bin
    }
    k_bin_bounds<<<(uint32_t)((n_aln + 1 + 255) / 256), 256, 0, s>>>(ctx->b[B_SKEY].as<uint32_t>(), (uint32_t)n_aln, n_bins + 2, d.bin_start);
    CK(cudaMemcpyAsync(ctx->h_status, d.st, sizeof(DevStatus), cudaMemcpyDeviceToHost, s));
    uint32_t* h_slots = reinterpret_cast<uint32_t*>(ctx->h_params);            // (pinned scratch; rewritten before every polish call)
    CK(cudaMemcpyAsync(h_slots, d.bin_start + n_bins + 1, 4, cudaMemcpyDeviceToHost, s));
    CK(cudaStreamSynchronize(s));
    CK(cudaGetLastError());
    ctx->max_ext = ctx->h_status->max_ext;
    const bool past_end = ctx->h_status->flags & FL_PAST_END;
    ctx->n_slots = *h_slots;
    const size_t ns = (size_t)ctx->n_slots + 16;
    CK(ctx->b[B_SREC].ensure(ns * sizeof(TileRec)));
    CK(ctx->b[B_SSEQ].ensure(BITS == 4 ? ns * TL_SEQ_QUADS * 16 + 256 : 256));
    CK(ctx->b[B_NK].ensure(ns * 16));
    CK(ctx->b[B_KF].ensure(na * 4));
    fill_data(ctx, d);
    if (ctx->n_slots) k_permute<<<(ctx->n_slots + 255) / 256, 256, 0, s>>>(d);
    if (seq_ready) { const int rc = seq_ready(); if (rc != PP_OK) return rc; }
    if (past_end)                                               // (alignments that start at or past their contig's end: rare)
        k_past_end<BITS><<<(uint32_t)std::min<uint64_t>((n_aln + 255) / 256, (uint64_t)ctx->sm_count * 16), 256, 0, s>>>(d);
    if (ctx->n_slots) {
        if (BITS == 4) {
            k_permute_seq<<<(ctx->n_slots + 255) / 256, 256, 0, s>>>(d);
        }
    }
    {   // tiles by decreasing slot count (the persistent kernel hands them out in that order)
        const uint32_t n_tiles = d.n_tiles;
        CK(ctx->b[B_TILEORDER].ensure(((size_t)n_tiles + 4) * 4));
        CK(ctx->b[B_KEY].ensure(((size_t)n_tiles + 4) * 8)); CK(ctx->b[B_VAL].ensure(((size_t)n_tiles + 4) * 4));
        uint32_t* w_in = ctx->b[B_KEY].as<uint32_t>();
        uint32_t* w_out = w_in + n_tiles + 2;
        uint32_t* idx_in = ctx->b[B_VAL].as<uint32_t>();
        fill_data(ctx, d);
        k_tile_weight<<<(n_tiles + 255) / 256, 256, 0, s>>>(d, w_in, idx_in);
        size_t tb = 0;
        CK(cub::DeviceRadixSort::SortPairsDescending(nullptr, tb, (const uint32_t*)nullptr, (uint32_t*)nullptr, (const uint32_t*)nullptr, (uint32_t*)nullptr, (int)n_tiles, 0, 32, s));
        CK(ctx->b[B_CUBTMP].ensure(tb + 256));
        tb = ctx->b[B_CUBTMP].cap;
        CK(cub::DeviceRadixSort::SortPairsDescending(ctx->b[B_CUBTMP].p, tb, w_in, w_out, idx_in, ctx->b[B_TILEORDER].as<uint32_t>(), (int)n_tiles, 0, 32, s));
    }
    CK(cudaStreamSynchronize(s));
    CK(cudaGetLastError());
    // the SAM-order scratch of the binning is not needed again; small ones stay for the next dataset (pp_polish per batch: no
    // cudaMalloc / cudaFree on the path)
    if (ctx->b[B_RECS].cap + ctx->b[B_KEY].cap + ctx->b[B_VAL].cap + ctx->b[B_SKEY].cap > (1ull << 30)) {
        ctx->b[B_RECS].release(); ctx->b[B_KEY].release(); ctx->b[B_VAL].release(); ctx->b[B_SKEY].release();
    }
    return PP_OK;
}

// seq_bits == 2 uploads (pp_alignments_to_2bit): 8 bytes of 2-bit codes -> the 16 bytes of one-hot BAM nibbles (A=1 C=2 G=4 T=8) the
// kernels read.  One thread per 32-base block; the tail of a read's last block expands to 'A's, which nothing reads (every consumer
// masks by the read length).
__device__ __forceinline__ unsigned long long expand16(uint32_t v) {
    unsigned long long x = v;
    x = (x | (x << 16)) & 0x0000FFFF0000FFFFull;
    x = (x | (x << 8)) & 0x00FF00FF00FF00FFull;
    x = (x | (x << 4)) & 0x0F0F0F0F0F0F0F0Full;
    x = (x | (x << 2)) & 0x3333333333333333ull;                 // code c of base i in bits 4i..4i+1
    const unsigned long long one = 0x1111111111111111ull;
    const unsigned long long b0 = x & one, b1 = (x >> 1) & one, n0 = b0 ^ one, n1 = b1 ^ one;
    return (n1 & n0) | ((n1 & b0) << 1) | ((b1 & n0) << 2) | ((b1 & b0) << 3);
}
__global__ void k_expand2(const uint2* __restrict__ in, uint4* __restrict__ out, uint64_t n_blocks) {
    for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < n_blocks; i += (uint64_t)gridDim.x * blockDim.x) {
        const uint2 v = __ldg(in + i);
        const unsigned long long lo = expand16(v.x), hi = expand16(v.y);
        out[i] = make_uint4((uint32_t)lo, (uint32_t)(lo >> 32), (uint32_t)hi, (uint32_t)(hi >> 32));
    }
}
// seq_bits == 2 uploads may leave cigar_off / read_id at home (pp_abi.h): prefix sums on the device.
__global__ void k_scan_inputs(const uint16_t* __restrict__ n_cigar, const uint8_t* __restrict__ flags, uint32_t* __restrict__ cigar_off,
                              uint32_t* __restrict__ read_id, uint64_t n) {         // (null = that array came with the batch)
    for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) {
        if (cigar_off) cigar_off[i] = n_cigar[i];
        if (read_id) read_id[i] = (flags[i] >> 7) & 1u;
    }
}
__global__ void k_ids_from_scan(uint32_t* __restrict__ read_id, uint64_t n) {      // inclusive count of group starts -> dense group id
    for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) {
        const uint32_t v = read_id[i];
        read_id[i] = v ? v - 1u : 0u;       // (records before the first PP_FLAG_NEWGROUP - a batch the packer did not make - join group 0: never an id of -1)
    }
}

// PP_FLAG_ESC records: their sequences sit behind the expanded pool.
__global__ void k_esc_offsets(uint32_t* __restrict__ seq_off, const uint8_t* __restrict__ flags, uint64_t n_aln, uint32_t first_esc_block) {
    for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < n_aln; i += (uint64_t)gridDim.x * blockDim.x)
        if (flags[i] & PP_FLAG_ESC) seq_off[i] += first_esc_block;
}

// The alignment arrays in ctx->b[B_CONTIG..B_SEQPOOL] become the resident dataset.
static int commit_dataset(pp_ctx* ctx, uint64_t n_aln, uint64_t n_reads, uint64_t n_ops, uint64_t seq_bytes, uint32_t seq_bits,
                          const std::function<int()>& seq_ready);
int pp_ctx_commit_dataset(pp_ctx* ctx, uint64_t n_aln, uint64_t n_reads, uint64_t n_ops, uint64_t seq_bytes, uint32_t seq_bits) {
    return commit_dataset(ctx, n_aln, n_reads, n_ops, seq_bytes, seq_bits, nullptr);
}
static int commit_dataset(pp_ctx* ctx, uint64_t n_aln, uint64_t n_reads, uint64_t n_ops, uint64_t seq_bytes, uint32_t seq_bits,
                          const std::function<int()>& seq_ready) {
    if (n_aln >= 0x7FFFFFFFull - 4096) return ctx->fail(PP_ERR_ARG, "more than 2^31-4096 alignments in one call");
    ctx->n_aln = n_aln; ctx->n_reads = n_reads; ctx->n_ops = n_ops; ctx->seq_bytes = seq_bytes; ctx->seq_bits = seq_bits;
    // first guesses; a call that overflows one of them grows it and repeats itself
    ctx->node_cap = (uint32_t)std::min<uint64_t>(0x7FFFFFFFull, std::max<uint64_t>(1 << 16, n_aln / 8 + ctx->G / 64));
    ctx->out_cap = ctx->G + ctx->G / 16 + (1u << 20);
    ctx->global_k = false;
    int rc = ctx->seq_bits == 4 ? bin_dataset<4>(ctx, seq_ready) : bin_dataset<8>(ctx, seq_ready);
    if (rc != PP_OK) return rc;
    ctx->have_ds = true;
    return PP_OK;
}

extern "C" int pp_dataset_upload(pp_ctx* ctx, const pp_contigs* c, const pp_alignments* a) {
    if (!ctx) return PP_ERR_ARG;
    if (!c || !a || !c->off || !c->bases || c->n_contigs == 0) return ctx->fail(PP_ERR_ARG, "pp_dataset_upload: null or empty contigs");
    const bool derive_ok = a->seq_bits == 2;                      // (the 2-bit wire format may leave cigar_off / read_id to the device)
    if (a->n_aln && (!a->contig || !a->ref_start || (!a->read_id && !derive_ok) || !a->seq_off || !a->seq_len || (!a->cigar_off && !derive_ok) ||
                     !a->n_cigar || !a->nm || !a->flags || !a->cigar_ops))
        return ctx->fail(PP_ERR_ARG, "pp_dataset_upload: null alignment array");
    if (a->seq_bits != 4 && a->seq_bits != 8 && a->seq_bits != 2) return ctx->fail(PP_ERR_ARG, "pp_dataset_upload: seq_bits must be 4, 8 or 2");
    const bool two_bit = a->seq_bits == 2;
    if (two_bit && ((a->seq_pool_bytes & 7) || (a->esc_pool_bytes & 15) || (a->esc_pool_bytes && !a->esc_pool) ||
                    a->seq_pool_bytes / 8 + a->esc_pool_bytes / 16 >= 0xFFFFFFFFull))
        return ctx->fail(PP_ERR_ARG, "pp_dataset_upload: 2-bit pool must be whole 8-byte blocks, esc_pool whole 16-byte blocks");
    if (a->n_aln >= 0x7FFFFFFFull - 4096) return ctx->fail(PP_ERR_ARG, "pp_dataset_upload: more than 2^31-4096 alignments in one call");
    CK(cudaSetDevice(ctx->device));
    ctx->have_ds = false;
    int rc;
    const void* host[DS_N];
    ds_host(a, host);
    const uint64_t cnt[3] = {a->n_aln, a->n_cigar_ops, 0};
    for (int k = 0; k < DS_SEQPOOL; ++k) {                                          // (the sequence pool follows below)
        const size_t bytes = ds_bytes(k, cnt, 0);
        CK(ctx->b[B_CONTIG + k].ensure(bytes + 64));
        const bool derived = !host[k] && (B_CONTIG + k == B_READID || B_CONTIG + k == B_CIGOFF);   // (rebuilt on the device below)
        if (bytes && !derived) CK(cudaMemcpyAsync(ctx->b[B_CONTIG + k].p, host[k], bytes, cudaMemcpyHostToDevice, ctx->stream));
    }
    if (a->n_aln && (!a->cigar_off || !a->read_id)) {
        const uint32_t grid = (uint32_t)std::min<uint64_t>((a->n_aln + 255) / 256, (uint64_t)ctx->sm_count * 32);
        uint32_t* co = a->cigar_off ? nullptr : ctx->b[B_CIGOFF].as<uint32_t>();
        uint32_t* ri = a->read_id ? nullptr : ctx->b[B_READID].as<uint32_t>();
        k_scan_inputs<<<grid, 256, 0, ctx->stream>>>(ctx->b[B_NCIG].as<uint16_t>(), ctx->b[B_FLAGS].as<uint8_t>(), co, ri, a->n_aln);
        size_t tb = 0;
        CK(cub::DeviceScan::InclusiveSum(nullptr, tb, (const uint32_t*)nullptr, (uint32_t*)nullptr, (int64_t)a->n_aln, ctx->stream));
        CK(ctx->b[B_CUBTMP].ensure(tb + 256));
        if (co) { tb = ctx->b[B_CUBTMP].cap; CK(cub::DeviceScan::ExclusiveSum(ctx->b[B_CUBTMP].p, tb, co, co, (int64_t)a->n_aln, ctx->stream)); }
        if (ri) {
            tb = ctx->b[B_CUBTMP].cap;
            CK(cub::DeviceScan::InclusiveSum(ctx->b[B_CUBTMP].p, tb, ri, ri, (int64_t)a->n_aln, ctx->stream));
            k_ids_from_scan<<<grid, 256, 0, ctx->stream>>>(ri, a->n_aln);
        }
    }
    if ((rc = pp_ctx_upload_contigs(ctx, c))) { ctx->err = "pp_dataset_upload: " + ctx->err; return rc; }
    // The sequence pool - two thirds of the bytes - goes last, on its own stream: the binning of the records (k_bin, the sort, k_permute)
    // needs none of it and runs while it crosses PCIe; the stream joins right before k_permute_seq.
    const uint64_t n_blocks2 = a->seq_pool_bytes / 8;
    const uint64_t seq_bytes = two_bit ? n_blocks2 * 16 + a->esc_pool_bytes : a->seq_pool_bytes;
    CK(ctx->b[B_SEQPOOL].ensure(seq_bytes + 256));
    if (two_bit) CK(ctx->b[B_SEQ2].ensure(a->seq_pool_bytes + 256));
    CK(cudaEventRecord(ctx->ev_small, ctx->stream));
    CK(cudaStreamWaitEvent(ctx->copy_stream, ctx->ev_small, 0));                   // (after the small arrays: they are needed first)
    if (!two_bit) {
        if (a->seq_pool_bytes) CK(cudaMemcpyAsync(ctx->b[B_SEQPOOL].p, a->seq_pool, a->seq_pool_bytes, cudaMemcpyHostToDevice, ctx->copy_stream));
    } else {
        if (a->seq_pool_bytes) CK(cudaMemcpyAsync(ctx->b[B_SEQ2].p, a->seq_pool, a->seq_pool_bytes, cudaMemcpyHostToDevice, ctx->copy_stream));
        if (a->esc_pool_bytes)
            CK(cudaMemcpyAsync(ctx->b[B_SEQPOOL].as<uint8_t>() + n_blocks2 * 16, a->esc_pool, a->esc_pool_bytes, cudaMemcpyHostToDevice, ctx->copy_stream));
        if (a->esc_pool_bytes && a->n_aln)
            k_esc_offsets<<<(uint32_t)std::min<uint64_t>((a->n_aln + 255) / 256, (uint64_t)ctx->sm_count * 32), 256, 0, ctx->stream>>>(
                ctx->b[B_SEQOFF].as<uint32_t>(), ctx->b[B_FLAGS].as<uint8_t>(), a->n_aln, (uint32_t)n_blocks2);
    }
    CK(cudaEventRecord(ctx->ev_seq, ctx->copy_stream));
    auto seq_ready = [&]() -> int {
        CK(cudaStreamWaitEvent(ctx->stream, ctx->ev_seq, 0));
        if (two_bit && n_blocks2)
            k_expand2<<<(uint32_t)std::min<uint64_t>((n_blocks2 + 255) / 256, (uint64_t)ctx->sm_count * 32), 256, 0, ctx->stream>>>(
                ctx->b[B_SEQ2].as<uint2>(), ctx->b[B_SEQPOOL].as<uint4>(), n_blocks2);
        return PP_OK;
    };
    rc = commit_dataset(ctx, a->n_aln, a->n_reads, a->n_cigar_ops, seq_bytes, two_bit ? 4u : a->seq_bits, seq_ready);
    if (rc != PP_OK) cudaStreamSynchronize(ctx->copy_stream);                      // (the caller's buffers are free again on every return)
    return rc;
}

static const char* err_text(unsigned code) {
    switch (code) {
        case ERR_UNKNOWN_CONTIG: return "query name in SAM but not in assembly";
        case ERR_SEQ_MISMATCH: return "CIGAR string does not match read sequence";
        case ERR_BAD_OP: return "unexpected character (other than M, =, X, I or D) in CIGAR string - did you use BWA MEM to generate your alignments?";
        case ERR_OOB: return "alignment extends past the end of its reference sequence";
        case ERR_NOSEQ: return "no alignments for read contain sequence";
        default: return "unknown device-side error";
    }
}

// --status-bed: k_tile's status bytes, padded to whole CTAs of k_status_heads / k_status_runs (which load 16 elements per thread); the
// depth keys are padded the same way (depth_key_bytes)
static size_t status_bytes(uint64_t G) { return (size_t)((G + SR_CHUNK - 1) / SR_CHUNK) * SR_CHUNK + 16; }

// A call's status bytes or depth keys -> the runs of report r, sized from their count.
template <class T>
static int report_runs(pp_ctx* ctx, const T* e, RunReport& r) {
    cudaStream_t s = ctx->stream;
    const uint32_t G = (uint32_t)ctx->G, n_blk = (uint32_t)((ctx->G + SR_CHUNK - 1) / SR_CHUNK);
    CK(ctx->b[B_RUNFIRST].ensure(((size_t)n_blk + 1) * 4));
    uint32_t* first = ctx->b[B_RUNFIRST].as<uint32_t>();
    CK(cudaMemsetAsync(first + n_blk, 0, 4, s));
    if (n_blk) k_status_heads<T><<<n_blk, SR_THREADS, 0, s>>>(e, G, first);
    size_t tb = 0;
    CK(cub::DeviceScan::ExclusiveSum(nullptr, tb, first, first, (int)n_blk + 1, s));
    CK(ctx->b[B_CUBTMP].ensure(tb + 256));
    tb = ctx->b[B_CUBTMP].cap;
    CK(cub::DeviceScan::ExclusiveSum(ctx->b[B_CUBTMP].p, tb, first, first, (int)n_blk + 1, s));
    uint32_t n = 0;
    CK(cudaMemcpyAsync(&n, first + n_blk, 4, cudaMemcpyDeviceToHost, s));
    CK(cudaStreamSynchronize(s));
    CK(cudaGetLastError());
    CK(ctx->b[r.b_start].ensure((size_t)n * 4 + 4)); CK(ctx->b[r.b_value].ensure((size_t)n * sizeof(T) + 8));
    if (n_blk) k_status_runs<T><<<n_blk, SR_THREADS, 0, s>>>(e, G, first, ctx->b[r.b_start].as<uint32_t>(), ctx->b[r.b_value].as<T>());
    CK(cudaGetLastError());
    ctx->launches += 2;
    r.n = n;
    r.have = true;
    return PP_OK;
}

// The k_tile instance that records what is asked for (CHG change list, STS status bytes, DEP depth keys).
using TileKernel = void (*)(DevData, VoteParams);
template <int BITS> static TileKernel tile_kernel(bool chg, bool sts, bool dep) {
    static const TileKernel k[8] = {k_tile<BITS, false, false, false>, k_tile<BITS, false, false, true>, k_tile<BITS, false, true, false>,
                                    k_tile<BITS, false, true, true>, k_tile<BITS, true, false, false>, k_tile<BITS, true, false, true>,
                                    k_tile<BITS, true, true, false>, k_tile<BITS, true, true, true>};
    return k[(chg ? 4 : 0) + (sts ? 2 : 0) + (dep ? 1 : 0)];
}

template <int BITS>
static int run_polish(pp_ctx* ctx, const pp_polish_params* prm, pp_polish_result* res) {
    cudaStream_t s = ctx->stream;
    const uint64_t G = ctx->G, n_aln = ctx->n_aln;
    const uint32_t n_tiles = (uint32_t)((G + TL_T - 1) / TL_T);              // = vote / compaction chunks
    const size_t padG = (size_t)n_tiles * TL_T + 16;                          // k_tile / k_compact move whole chunks with vector accesses
    ctx->have_changes = ctx->status.have = ctx->depth.have = false;

    CK(ctx->b[B_OUTOFF].ensure(((size_t)ctx->n_contigs + 1) * 8));
    CK(ctx->b[B_RES].ensure(padG * 2)); CK(ctx->b[B_RECAT].ensure((G + 1) * 4)); CK(ctx->b[B_CHUNKDELTA].ensure((size_t)n_tiles * 8));
    CK(ctx->b[B_PARAMS].ensure(sizeof(DevParams)));
    if (!ctx->tile_attr_set) {
        for (int i = 0; i < 8; ++i) {
            CK(cudaFuncSetAttribute(tile_kernel<4>(i & 4, i & 2, i & 1), cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(TileShared)));
            CK(cudaFuncSetAttribute(tile_kernel<8>(i & 4, i & 2, i & 1), cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(TileShared)));
        }
        ctx->tile_attr_set = true;
    }

    ctx->h_params->fv = prm->fraction_valid; ctx->h_params->fi = prm->fraction_invalid;
    ctx->h_params->min_depth = prm->min_depth; ctx->h_params->max_errors = prm->max_errors;
    ctx->h_params->careful = prm->careful ? 1 : 0; ctx->h_params->pad = 0;

    for (int attempt = 0; attempt < 8; ++attempt) {
        const uint32_t node_cap = ctx->node_cap;
        const uint64_t out_cap = ctx->out_cap;
        // everything that must be zero at the start of a call lives in one small pool: one memset (the counters live in shared
        // memory, and the 4 B per position of chain heads are zeroed tile by tile inside k_tile)
        size_t zoff = 0;
        auto carve = [&](size_t bytes) { size_t o = zoff; zoff += (bytes + 255) & ~size_t(255); return o; };
        const size_t o_chg = carve((size_t)ctx->n_contigs * 8), o_zero = carve((size_t)ctx->n_contigs * 8),
                     o_tdep = carve((size_t)ctx->n_contigs * 8), o_status = carve(sizeof(DevStatus)),
                     o_k = carve(ctx->global_k ? (ctx->n_reads + 1) * 4 : 4), o_prm = carve(sizeof(DevParams));
        const bool one_copy = zoff <= PP_INIT_IMAGE;         // (not with thousands of contigs or the global-k fallback: then memsets)
        CK(ctx->b[B_ZEROPOOL].ensure(zoff));
        CK(ctx->b[B_HEADS].ensure(padG * 4 + 64));
        uint8_t* zp = ctx->b[B_ZEROPOOL].as<uint8_t>();
        CK(ctx->b[B_NODES].ensure((size_t)node_cap * sizeof(OthNode)));
        CK(ctx->b[B_OUT].ensure(out_cap + 64));
        // --depth-bedgraph / --status-bed: the depth keys, then the status bytes, in one buffer (VoteParams::sts), allocated before the
        // timed stages
        const size_t key_bytes = ctx->depth.on ? depth_key_bytes(G) : 0;
        if (ctx->status.on || ctx->depth.on) CK(ctx->b[B_STS].ensure(key_bytes + (ctx->status.on ? status_bytes(G) : 16)));

        DevData d;
        fill_data(ctx, d);
        d.k = (uint32_t*)(zp + o_k);
        d.oth_head = ctx->b[B_HEADS].as<uint32_t>(); d.nodes = ctx->b[B_NODES].as<OthNode>(); d.node_cap = node_cap;
        d.prm = one_copy ? (DevParams*)(zp + o_prm) : ctx->b[B_PARAMS].as<DevParams>();
        d.st = (DevStatus*)(zp + o_status);
        ctx->launches = 0;

        // ---- stage 0: reset
        CK(cudaEventRecord(ctx->ev[0], s));
        if (one_copy) {                                      // zeros, the options and "no error" in one host-to-device copy
            memset(ctx->h_init, 0, zoff);
            memcpy(ctx->h_init + o_prm, ctx->h_params, sizeof(DevParams));
            memset(ctx->h_init + o_status + offsetof(DevStatus, err), 0xFF, 8);
            CK(cudaMemcpyAsync(zp, ctx->h_init, zoff, cudaMemcpyHostToDevice, s));
        } else {
            CK(cudaMemcpyAsync(ctx->b[B_PARAMS].p, ctx->h_params, sizeof(DevParams), cudaMemcpyHostToDevice, s));
            CK(cudaMemsetAsync(zp, 0, zoff, s));
            CK(cudaMemsetAsync(&d.st->err, 0xFF, 8, s));
        }
        // ---- stage 1: (fallback only) global k of multi-record groups
        CK(cudaEventRecord(ctx->ev[1], s));
        if (n_aln && ctx->global_k) {
            k_classify_multi<<<(uint32_t)std::min<uint64_t>((n_aln + 255) / 256, (uint64_t)ctx->sm_count * 8), 256, 0, s>>>(d);
            ctx->launches++;
        }
        // ---- stage 2: goodness / k of every alignment under these options (SAM order, coalesced)
        CK(cudaEventRecord(ctx->ev[2], s));
        if (n_aln) {
            const uint32_t grid = (uint32_t)std::min<uint64_t>((n_aln + PR_THREADS - 1) / PR_THREADS, (uint64_t)ctx->sm_count * 8);
            if (ctx->global_k) k_goodk<true><<<grid, PR_THREADS, 0, s>>>(d);
            else k_goodk<false><<<grid, PR_THREADS, 0, s>>>(d);
            ctx->launches++;
        }
        // ---- stage 3: scatter + ordered depth + vote, one tile of positions at a time, counters in shared memory
        CK(cudaEventRecord(ctx->ev[3], s));
        VoteParams vp;
        vp.n_chunks = n_tiles;
        vp.out = ctx->b[B_OUT].as<uint8_t>(); vp.out_cap = out_cap;
        vp.out_off = ctx->b[B_OUTOFF].as<unsigned long long>();
        vp.changed = (unsigned long long*)(zp + o_chg); vp.zero_depth = (unsigned long long*)(zp + o_zero); vp.total_depth = (double*)(zp + o_tdep);
        vp.res = ctx->b[B_RES].as<uint16_t>(); vp.rec_at = ctx->b[B_RECAT].as<uint32_t>();
        vp.chunk_delta = ctx->b[B_CHUNKDELTA].as<long long>();
        vp.dbg = nullptr;
        if (ctx->debug_on) { CK(ctx->b[B_DEBUG].ensure((G + 1) * sizeof(pp_debug_pos))); vp.dbg = ctx->b[B_DEBUG].as<pp_debug_pos>(); }
        vp.chg = nullptr; vp.chg_pos = nullptr; vp.chg_n = &d.st->n_changes; vp.chg_cap = 0;
        if (ctx->changes_on) {
            if (ctx->chg_cap == 0) ctx->chg_cap = (uint32_t)std::max<uint64_t>(4096, G / 256);
            CK(ctx->b[B_CHG].ensure((size_t)ctx->chg_cap * sizeof(pp_debug_pos))); CK(ctx->b[B_CHGPOS].ensure((size_t)ctx->chg_cap * 4));
            vp.chg = ctx->b[B_CHG].as<pp_debug_pos>(); vp.chg_pos = ctx->b[B_CHGPOS].as<uint32_t>(); vp.chg_cap = ctx->chg_cap;
        }
        vp.sts = (ctx->status.on || ctx->depth.on) ? ctx->b[B_STS].as<uint8_t>() : nullptr;
        {
            const TileKernel kt = tile_kernel<BITS>(vp.chg, ctx->status.on, ctx->depth.on);
            int occ = 1;
            CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, kt, TL_THREADS, sizeof(TileShared)));
            const uint32_t grid = std::min<uint32_t>(n_tiles, (uint32_t)ctx->sm_count * (uint32_t)std::max(occ, 1));   // persistent: tiles by ticket
            kt<<<grid, TL_THREADS, sizeof(TileShared), s>>>(d, vp);
            ctx->launches++;
        }
        // ---- stage 4: compaction
        CK(cudaEventRecord(ctx->ev[4], s));
        k_compact<BITS><<<n_tiles, VT_THREADS, 0, s>>>(d, vp);
        ctx->launches++;
        CK(cudaEventRecord(ctx->ev[5], s));
        CK(cudaMemcpyAsync(ctx->h_status, d.st, sizeof(DevStatus), cudaMemcpyDeviceToHost, s));
        CK(cudaStreamSynchronize(s));
        CK(cudaGetLastError());
        const DevStatus hs = *ctx->h_status;
#ifdef PP_TILE_PROF
        fprintf(stderr, "[tile prof] tiles %llu; cycles/tile: A %.0f B %.0f queue %.0f C %.0f D+E %.0f; queued reads/tile %.1f (max %llu); "
                "chunk wait/tile/warp %.0f\n", hs.prof[6],
                (double)hs.prof[0] / hs.prof[6], (double)hs.prof[1] / hs.prof[6], (double)hs.prof[2] / hs.prof[6], (double)hs.prof[3] / hs.prof[6],
                (double)hs.prof[4] / hs.prof[6], (double)hs.prof[5] / hs.prof[6], hs.prof[7], (double)hs.prof[11] / hs.prof[6] / (TL_THREADS / 32));
        fprintf(stderr, "[tile prof] depth walks %llu (%.2f per tile, %llu tiles with one), %.0f cycles each\n", hs.prof[9], (double)hs.prof[9] / hs.prof[6], hs.prof[10],
                hs.prof[9] ? (double)hs.prof[8] / hs.prof[9] : 0.0);
        {   // what the chunk loop streams per call, by array, from the slots the tiles scanned (look-back bins included)
            const double sl = (double)hs.prof[12], t = (double)hs.prof[6];
            fprintf(stderr, "[tile prof] slots scanned %llu; MB: records %.1f bases %.1f kf %.1f wrec %.1f draft+verdicts+chain heads %.1f\n",
                    hs.prof[12], sl * sizeof(TileRec) / 1e6, BITS == 4 ? sl * 16 * TL_SEQ_QUADS / 1e6 : 0.0, sl * 4 / 1e6, sl * 16 / 1e6,
                    t * (TL_T + 16 + 2 * TL_T + 4 * TL_T) / 1e6);
        }
#endif
        if (hs.err != ~0ull) {
            res->error_aln = (int64_t)(hs.err >> 8);
            return ctx->fail(PP_ERR_INPUT, std::string(err_text((unsigned)(hs.err & 0xFF))) + " (alignment " + std::to_string(hs.err >> 8) + ")");
        }
        // a side buffer was too small or a read group too large for the in-kernel scan: grow / switch mode and repeat
        bool again = false;
        if (hs.flags & FL_BIGGROUP) { if (ctx->global_k) return ctx->fail(PP_ERR_CUDA, "internal error: FL_BIGGROUP in global-k mode"); ctx->global_k = true; again = true; }
        if (hs.flags & FL_NODE_OVF) { ctx->node_cap = (uint32_t)std::min<uint64_t>(0x7FFFFFFFull, (uint64_t)hs.node_count + hs.node_count / 4 + 1024); again = true; }
        if (!again && (hs.flags & FL_OUT_OVF)) { ctx->out_cap = hs.out_len + 64; again = true; }
        // the change list: its exact length is the number of changed positions, counted past the end (= the sum of `changed`)
        if (!again && ctx->changes_on && hs.n_changes > ctx->chg_cap) { ctx->chg_cap = hs.n_changes; again = true; }
        if (again) continue;

        ctx->have_debug = ctx->debug_on; ctx->last_head = d.oth_head; ctx->last_nodes = std::min(hs.node_count, node_cap);
        ctx->have_changes = ctx->changes_on; ctx->n_changes = ctx->changes_on ? hs.n_changes : 0; ctx->chg_pool = -1;
        if (ctx->status.on) {
            const int rc = report_runs(ctx, vp.sts + key_bytes, ctx->status);
            if (rc != PP_OK) return rc;
        }
        if (ctx->depth.on) {
            const int rc = report_runs(ctx, reinterpret_cast<const unsigned long long*>(vp.sts), ctx->depth);
            if (rc != PP_OK) return rc;
        }
        res->out_len = hs.out_len;
        res->n_aln_used = hs.n_used;
        res->error_aln = -1;
        memset(&res->timing, 0, sizeof res->timing);
        float ms;
        CK(cudaEventElapsedTime(&ms, ctx->ev[0], ctx->ev[1])); res->timing.stage_ms[0] = ms;
        CK(cudaEventElapsedTime(&ms, ctx->ev[1], ctx->ev[2])); res->timing.stage_ms[1] = ms;
        CK(cudaEventElapsedTime(&ms, ctx->ev[2], ctx->ev[3])); res->timing.stage_ms[2] = ms;
        CK(cudaEventElapsedTime(&ms, ctx->ev[3], ctx->ev[4])); res->timing.stage_ms[3] = ms;
        CK(cudaEventElapsedTime(&ms, ctx->ev[4], ctx->ev[5])); res->timing.stage_ms[4] = ms;
        CK(cudaEventElapsedTime(&ms, ctx->ev[0], ctx->ev[5])); res->timing.total_ms = ms;
        res->timing.launches = ctx->launches;

        if (res->out_bases) {
            if (res->out_cap < hs.out_len) return ctx->fail(PP_ERR_ARG, "out_cap too small: need " + std::to_string(hs.out_len) + " bytes");
            CK(cudaEventRecord(ctx->ev[7], s));
            CK(cudaMemcpyAsync(res->out_bases, vp.out, hs.out_len, cudaMemcpyDeviceToHost, s));
            if (res->out_off) CK(cudaMemcpyAsync(res->out_off, vp.out_off, ((size_t)ctx->n_contigs + 1) * 8, cudaMemcpyDeviceToHost, s));
            if (res->changed) CK(cudaMemcpyAsync(res->changed, vp.changed, (size_t)ctx->n_contigs * 8, cudaMemcpyDeviceToHost, s));
            if (res->zero_depth) CK(cudaMemcpyAsync(res->zero_depth, vp.zero_depth, (size_t)ctx->n_contigs * 8, cudaMemcpyDeviceToHost, s));
            if (res->total_depth) CK(cudaMemcpyAsync(res->total_depth, vp.total_depth, (size_t)ctx->n_contigs * 8, cudaMemcpyDeviceToHost, s));
            CK(cudaEventRecord(ctx->ev[8], s));
            CK(cudaStreamSynchronize(s));
            CK(cudaEventElapsedTime(&ms, ctx->ev[7], ctx->ev[8]));
            res->timing.stage_ms[7] = ms;
        }
        return PP_OK;
    }
    return ctx->fail(PP_ERR_NOMEM, "side buffers kept overflowing");
}

static int check_params(pp_ctx* ctx, const pp_polish_params* p) {
    if (!p) return ctx->fail(PP_ERR_ARG, "null params");
    // polish.rs:277-287 (the same text the reference prints)
    if (!(p->fraction_valid > 0.0 && p->fraction_valid < 1.0)) return ctx->fail(PP_ERR_INPUT, "--fraction_valid must be between 0 and 1 (exclusive)");
    if (!(p->fraction_invalid > 0.0 && p->fraction_invalid < 1.0)) return ctx->fail(PP_ERR_INPUT, "--fraction_invalid must be between 0 and 1 (exclusive)");
    if (p->fraction_invalid >= p->fraction_valid) return ctx->fail(PP_ERR_INPUT, "--fraction_invalid must be less than --fraction_valid");
    return PP_OK;
}

extern "C" int pp_polish_resident(pp_ctx* ctx, const pp_polish_params* params, pp_polish_result* result) {
    if (!ctx) return PP_ERR_ARG;
    if (!result) return ctx->fail(PP_ERR_ARG, "null result");
    if (!ctx->have_ds) return ctx->fail(PP_ERR_ARG, "pp_polish_resident: no dataset uploaded");
    int rc = check_params(ctx, params);
    if (rc) return rc;
    CK(cudaSetDevice(ctx->device));
    result->error_aln = -1;
    return ctx->seq_bits == 4 ? run_polish<4>(ctx, params, result) : run_polish<8>(ctx, params, result);
}

extern "C" int pp_polish(pp_ctx* ctx, const pp_contigs* contigs, const pp_alignments* alns,
                         const pp_polish_params* params, pp_polish_result* result) {
    if (!ctx) return PP_ERR_ARG;
    if (!result) return ctx->fail(PP_ERR_ARG, "null result");
    int rc = check_params(ctx, params);
    if (rc) return rc;
    CK(cudaSetDevice(ctx->device));
    CK(cudaEventRecord(ctx->ev[9], ctx->stream));
    rc = pp_dataset_upload(ctx, contigs, alns);
    if (rc) return rc;
    CK(cudaEventRecord(ctx->ev[10], ctx->stream));
    CK(cudaEventSynchronize(ctx->ev[10]));
    float h2d = 0;
    CK(cudaEventElapsedTime(&h2d, ctx->ev[9], ctx->ev[10]));
    result->error_aln = -1;
    rc = ctx->seq_bits == 4 ? run_polish<4>(ctx, params, result) : run_polish<8>(ctx, params, result);
    if (rc == PP_OK) result->timing.stage_ms[6] = h2d;
    return rc;
}

extern "C" int pp_polish_set_debug(pp_ctx* ctx, int on) {
    if (!ctx) return PP_ERR_ARG;
    ctx->debug_on = on == 1;            // 2 = stop recording but keep the last call's records readable
    if (on == 0) ctx->have_debug = false;
    return PP_OK;
}

extern "C" int pp_polish_debug_fetch(pp_ctx* ctx, uint64_t first_pos, uint64_t n_pos, pp_debug_pos* out) {
    if (!ctx) return PP_ERR_ARG;
    if (!ctx->have_debug) return ctx->fail(PP_ERR_ARG, "pp_polish_debug_fetch: the last polish did not record debug positions (pp_polish_set_debug)");
    if (!out || first_pos + n_pos > ctx->G) return ctx->fail(PP_ERR_ARG, "pp_polish_debug_fetch: range outside the assembly");
    CK(cudaSetDevice(ctx->device));
    CK(cudaMemcpyAsync(out, ctx->b[B_DEBUG].as<pp_debug_pos>() + first_pos, n_pos * sizeof(pp_debug_pos), cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    return PP_OK;
}

extern "C" int pp_polish_debug_alleles(pp_ctx* ctx, uint32_t* head, pp_debug_node* nodes, uint64_t node_cap, uint64_t* n_nodes) {
    if (!ctx) return PP_ERR_ARG;
    if (!ctx->have_debug || !ctx->last_head) return ctx->fail(PP_ERR_ARG, "pp_polish_debug_alleles: no debug polish on this context");
    if (n_nodes) *n_nodes = ctx->last_nodes;
    if (!head && !nodes && node_cap == 0) return PP_ERR_ARG;       // size query
    if (!head || (ctx->last_nodes && !nodes) || node_cap < ctx->last_nodes) return ctx->fail(PP_ERR_ARG, "pp_polish_debug_alleles: buffers too small");
    static_assert(sizeof(pp_debug_node) == sizeof(OthNode), "debug node layout");
    CK(cudaSetDevice(ctx->device));
    CK(cudaMemcpyAsync(head, ctx->last_head, ctx->G * 4, cudaMemcpyDeviceToHost, ctx->stream));
    if (ctx->last_nodes) CK(cudaMemcpyAsync(nodes, ctx->b[B_NODES].p, (size_t)ctx->last_nodes * sizeof(OthNode), cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    return PP_OK;
}

// k_allele_strings over n rows of the last call (positions pos_dev, records rec_dev) into B_STRPOOL / B_STROFF; *bytes = pool bytes.
template <int BITS>
static int allele_strings(pp_ctx* ctx, const uint32_t* pos_dev, const pp_debug_pos* rec_dev, bool by_pos, uint32_t n, uint64_t* bytes) {
    cudaStream_t s = ctx->stream;
    OthCtx oc;
    oc.nodes = ctx->b[B_NODES].as<OthNode>(); oc.head = ctx->last_head;
    oc.sr = SeqRef{ctx->b[B_SEQPOOL].as<uint8_t>(), ctx->b[B_SEQOFF].as<uint32_t>(), ctx->b[B_SEQLEN].as<uint16_t>(), ctx->b[B_FLAGS].as<uint8_t>()};
    CK(ctx->b[B_STROFF].ensure((size_t)n * 8 + 8));
    unsigned long long* used = ctx->b[B_STROFF].as<unsigned long long>() + n;                 // (behind the offsets)
    uint64_t cap = std::max<uint64_t>(ctx->b[B_STRPOOL].cap, (uint64_t)n * 16 + 4096);
    for (int attempt = 0; attempt < 2; ++attempt) {
        CK(ctx->b[B_STRPOOL].ensure(cap));
        CK(cudaMemsetAsync(used, 0, 8, s));
        if (n) k_allele_strings<BITS><<<(n + 255) / 256, 256, 0, s>>>(oc, pos_dev, rec_dev, by_pos, n, ctx->b[B_STRPOOL].as<uint8_t>(), cap, used, ctx->b[B_STROFF].as<unsigned long long>());
        CK(cudaMemcpyAsync(bytes, used, 8, cudaMemcpyDeviceToHost, s));
        CK(cudaStreamSynchronize(s));
        CK(cudaGetLastError());
        if (*bytes <= cap) return PP_OK;
        cap = *bytes;                                                     // the exact size: the second round fits
    }
    return ctx->fail(PP_ERR_NOMEM, "allele strings: pool kept overflowing");
}
static int allele_strings(pp_ctx* ctx, const uint32_t* pos_dev, const pp_debug_pos* rec_dev, bool by_pos, uint32_t n, uint64_t* bytes) {
    return ctx->seq_bits == 4 ? allele_strings<4>(ctx, pos_dev, rec_dev, by_pos, n, bytes) : allele_strings<8>(ctx, pos_dev, rec_dev, by_pos, n, bytes);
}

// internal (host_api.cpp): the allele strings of the --debug records at n positions (pp_polish_set_debug), in k_allele_strings' format
int pp_polish_debug_strings(pp_ctx* ctx, const uint32_t* pos, uint32_t n, std::vector<uint64_t>& off, std::vector<uint8_t>& pool) {
    if (!ctx->have_debug || !ctx->last_head) return ctx->fail(PP_ERR_ARG, "pp_polish_debug_strings: no debug polish on this context");
    CK(cudaSetDevice(ctx->device));
    CK(ctx->b[B_STRPOS].ensure((size_t)n * 4 + 4));
    if (n) CK(cudaMemcpyAsync(ctx->b[B_STRPOS].p, pos, (size_t)n * 4, cudaMemcpyHostToDevice, ctx->stream));
    uint64_t bytes = 0;
    const int rc = allele_strings(ctx, ctx->b[B_STRPOS].as<uint32_t>(), ctx->b[B_DEBUG].as<pp_debug_pos>(), true, n, &bytes);
    if (rc != PP_OK) return rc;
    off.resize(n);
    pool.resize(bytes);
    if (n) CK(cudaMemcpyAsync(off.data(), ctx->b[B_STROFF].p, (size_t)n * 8, cudaMemcpyDeviceToHost, ctx->stream));
    if (bytes) CK(cudaMemcpyAsync(pool.data(), ctx->b[B_STRPOOL].p, bytes, cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    return PP_OK;
}

extern "C" int pp_polish_set_changes(pp_ctx* ctx, int on) {
    if (!ctx) return PP_ERR_ARG;
    ctx->changes_on = on == 1;          // 2 = stop recording but keep the last call's rows readable
    if (on == 0) ctx->have_changes = false;
    return PP_OK;
}

extern "C" int pp_polish_changes_fetch(pp_ctx* ctx, uint64_t row_cap, uint64_t* pos, pp_debug_pos* rows, uint64_t* pool_off, uint8_t* pool,
                                       uint64_t pool_cap, uint64_t* n_rows, uint64_t* pool_bytes) {
    if (!ctx) return PP_ERR_ARG;
    if (!ctx->have_changes || !ctx->last_head) return ctx->fail(PP_ERR_ARG, "pp_polish_changes_fetch: the last polish did not record changes (pp_polish_set_changes)");
    if (!n_rows || !pool_bytes) return ctx->fail(PP_ERR_ARG, "pp_polish_changes_fetch: null size pointers");
    CK(cudaSetDevice(ctx->device));
    const uint32_t n = ctx->n_changes;
    if (ctx->chg_pool < 0) {
        uint64_t bytes = 0;
        const int rc = allele_strings(ctx, ctx->b[B_CHGPOS].as<uint32_t>(), ctx->b[B_CHG].as<pp_debug_pos>(), false, n, &bytes);
        if (rc != PP_OK) return rc;
        ctx->chg_pool = (int64_t)bytes;
    }
    *n_rows = n;
    *pool_bytes = (uint64_t)ctx->chg_pool;
    if (row_cap == 0 && pool_cap == 0 && n > 0) return PP_OK;                                 // size query
    if (row_cap < n || pool_cap < *pool_bytes || (n && (!pos || !rows || !pool_off || !pool)))
        return ctx->fail(PP_ERR_ARG, "pp_polish_changes_fetch: buffers too small");
    // the rows arrive in the order the tiles appended them: sorted by position here, the pool stays as it is
    std::vector<uint32_t> p(n);
    std::vector<pp_debug_pos> r(n);
    std::vector<uint64_t> o(n);
    if (n) {
        CK(cudaMemcpyAsync(p.data(), ctx->b[B_CHGPOS].p, (size_t)n * 4, cudaMemcpyDeviceToHost, ctx->stream));
        CK(cudaMemcpyAsync(r.data(), ctx->b[B_CHG].p, (size_t)n * sizeof(pp_debug_pos), cudaMemcpyDeviceToHost, ctx->stream));
        CK(cudaMemcpyAsync(o.data(), ctx->b[B_STROFF].p, (size_t)n * 8, cudaMemcpyDeviceToHost, ctx->stream));
    }
    if (*pool_bytes) CK(cudaMemcpyAsync(pool, ctx->b[B_STRPOOL].p, *pool_bytes, cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    std::vector<uint32_t> order(n);
    for (uint32_t i = 0; i < n; ++i) order[i] = i;
    std::sort(order.begin(), order.end(), [&](uint32_t a, uint32_t b) { return p[a] < p[b]; });
    for (uint32_t i = 0; i < n; ++i) { pos[i] = p[order[i]]; rows[i] = r[order[i]]; pool_off[i] = o[order[i]]; }
    return PP_OK;
}

// pp_polish_set_status / pp_polish_set_depth: on = 1 records report r from the next call on; 2 stops recording but keeps the last
// call's runs readable; 0 forgets them.
static int set_runs(pp_ctx* ctx, RunReport& r, int on) {
    r.on = on == 1;
    if (on != 1) { CK(cudaSetDevice(ctx->device)); ctx->b[B_STS].release(); ctx->b[B_RUNFIRST].release(); }
    if (on == 0) { r.have = false; ctx->b[r.b_start].release(); ctx->b[r.b_value].release(); }
    return PP_OK;
}

// pp_polish_status_fetch / pp_polish_depth_fetch: the runs of report r, which the messages name `what` ("status" / "depth").
template <class T>
static int fetch_runs(pp_ctx* ctx, const RunReport& r, const char* what, uint64_t run_cap, uint64_t* start, T* value, uint64_t* n_runs) {
    const std::string fn = std::string("pp_polish_") + what + "_fetch";
    if (!r.have) return ctx->fail(PP_ERR_ARG, fn + ": the last polish did not record " + what + " (pp_polish_set_" + what + ")");
    if (!n_runs) return ctx->fail(PP_ERR_ARG, fn + ": null size pointer");
    const uint32_t n = r.n;
    *n_runs = n;
    if (run_cap == 0 && n > 0) return PP_OK;                                                   // size query
    if (run_cap < n || (n && (!start || !value))) return ctx->fail(PP_ERR_ARG, fn + ": buffers too small");
    CK(cudaSetDevice(ctx->device));
    std::vector<uint32_t> st(n);
    if (n) {
        CK(cudaMemcpyAsync(st.data(), ctx->b[r.b_start].p, (size_t)n * 4, cudaMemcpyDeviceToHost, ctx->stream));
        CK(cudaMemcpyAsync(value, ctx->b[r.b_value].p, (size_t)n * sizeof(T), cudaMemcpyDeviceToHost, ctx->stream));
    }
    CK(cudaStreamSynchronize(ctx->stream));
    std::copy(st.begin(), st.end(), start);
    return PP_OK;
}

extern "C" int pp_polish_set_status(pp_ctx* ctx, int on) { return ctx ? set_runs(ctx, ctx->status, on) : PP_ERR_ARG; }

extern "C" int pp_polish_status_fetch(pp_ctx* ctx, uint64_t run_cap, uint64_t* start, uint8_t* status, uint64_t* n_runs) {
    return ctx ? fetch_runs(ctx, ctx->status, "status", run_cap, start, status, n_runs) : PP_ERR_ARG;
}

extern "C" int pp_polish_set_depth(pp_ctx* ctx, int on) { return ctx ? set_runs(ctx, ctx->depth, on) : PP_ERR_ARG; }

extern "C" int pp_polish_depth_fetch(pp_ctx* ctx, uint64_t run_cap, uint64_t* start, uint64_t* tenths, uint64_t* n_runs) {
    return ctx ? fetch_runs(ctx, ctx->depth, "depth", run_cap, start, tenths, n_runs) : PP_ERR_ARG;
}
