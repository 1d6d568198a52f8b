// tok_kernels.cu — SAM text -> packed alignments ON THE DEVICE (SURVEY.md §8f-1, "GPU SAM tokeniser / packer").
//
// The text of one SAM file is streamed into HBM (pinned double buffers, several reader threads) and turned into exactly the
// arrays the host packer (sam_pack.cpp) would have produced, so that `polypolish polish` spends its time on PCIe instead
// of on a host parse:
//
//   k_tok_count   newlines per 16 KiB tile                                   text read once      (HBM-bound)
//   (cub scan)    tile offsets
//   k_tok_index   line starts                                                text read once
//   k_tok_parse   one thread per line: columns, FLAG/POS/NM/ZP, CIGAR check, RNAME -> contig     text read once
//   (cub scans)   alignment index, CIGAR-pool offset, sequence-pool offset of every line
//   k_tok_emit    one thread per aligned line: record arrays, CIGAR ops, 4-bit (or 8-bit) bases   CIGAR+SEQ read again
//   k_tok_heads   one thread per alignment: does it open a read group (QNAME compare with its predecessor)
//   (cub scan)    read ids
//   k_tok_groups  one thread per group head: SEQ="*" records take the group's source sequence
//
// Per-item logic lives in tok_line.h (host+device, CPU-tested against the host packer).  The host packer stays the
// authority on everything unusual: a malformed line, a limit, a group without sequence make the call return PP_TOK_HOST and
// the caller runs pp_pack_* on the same text, which yields the result or the reference's own error message
// (alignment.rs:49-98, 225-346).
#include <cuda_runtime.h>

#include <cub/block/block_reduce.cuh>
#include <cub/block/block_scan.cuh>
#include <cub/device/device_scan.cuh>

#include <fcntl.h>
#include <sys/mman.h>
#include <sys/stat.h>
#include <sys/statvfs.h>
#include <unistd.h>

#include <cerrno>
#include <algorithm>
#include <atomic>
#include <chrono>
#include <string>
#include <thread>
#include <vector>

#include "pp_ctx.cuh"
#include "tok_line.h"
#include "tok_table.h"
#include "tok_strip.h"

// A temporary that does not fit in device memory is not an error of the data: the host text code takes over.
#define TRY_ALLOC(x) do { if ((x) != cudaSuccess) { cudaGetLastError(); return PP_TOK_HOST; } } while (0)

namespace {

constexpr int TK_TILE = 16384;        // bytes of text per CTA in the newline passes
constexpr int TK_THREADS = 256;
constexpr int TK_LINE_THREADS = 128;  // threads (= lines) per CTA in the per-line passes
constexpr int TK_READERS = 16;        // at most this many host threads stream a file into the device
constexpr size_t TK_SLOT = 4u << 20;  // pinned bytes per slot (two slots per reader)
constexpr size_t TK_LOOK = 1u << 20;  // QUAL-stripping upload: how far past its nominal slice a reader looks for the line end

struct TokStatus {
    unsigned long long first_bad;     // smallest line index the device does not accept (~0 = none)
    unsigned int need8;               // a SEQ byte outside the 4-bit alphabet
    unsigned int group_err;           // a read group without any sequence (alignment.rs:319-321)
};

struct TokTable {                     // device pointers of the contig-name table and the nibble table
    tok::ContigTable ct;
    const uint8_t* nibtab;
};

__device__ __forceinline__ uint32_t newline_mask(uint32_t w) { return __vcmpeq4(w, 0x0A0A0A0Au); }

__global__ void __launch_bounds__(TK_THREADS) k_tok_count(const uint8_t* __restrict__ text, uint64_t n16, unsigned long long* __restrict__ tile_cnt) {
    const uint64_t t0 = (uint64_t)blockIdx.x * TK_TILE;
    uint32_t c = 0;
    for (uint32_t off = threadIdx.x * 16; off < TK_TILE; off += TK_THREADS * 16) {
        const uint64_t p = t0 + off;
        if (p < n16) {
            const uint4 v = __ldg(reinterpret_cast<const uint4*>(text + p));
            c += __popc(newline_mask(v.x) & 0x01010101u) + __popc(newline_mask(v.y) & 0x01010101u) +
                 __popc(newline_mask(v.z) & 0x01010101u) + __popc(newline_mask(v.w) & 0x01010101u);
        }
    }
    typedef cub::BlockReduce<uint32_t, TK_THREADS> BR;
    __shared__ typename BR::TempStorage tmp;
    const uint32_t s = BR(tmp).Sum(c);
    if (threadIdx.x == 0) tile_cnt[blockIdx.x] = s;
}

// line_start[i] = offset of the first byte of line i; line_start[0] = 0, line_start[k+1] = position after newline k.
__global__ void __launch_bounds__(TK_THREADS) k_tok_index(const uint8_t* __restrict__ text, uint64_t n16, const unsigned long long* __restrict__ tile_off,
                                                          unsigned long long* __restrict__ line_start) {
    typedef cub::BlockScan<uint32_t, TK_THREADS> BS;
    __shared__ typename BS::TempStorage tmp;
    const uint64_t t0 = (uint64_t)blockIdx.x * TK_TILE;
    unsigned long long run = tile_off[blockIdx.x];
    if (blockIdx.x == 0 && threadIdx.x == 0) line_start[0] = 0;
    for (uint32_t it = 0; it < TK_TILE / (TK_THREADS * 16); ++it) {
        const uint64_t p = t0 + (uint64_t)it * TK_THREADS * 16 + threadIdx.x * 16;
        uint32_t m[4] = {0, 0, 0, 0};
        if (p < n16) {
            const uint4 v = __ldg(reinterpret_cast<const uint4*>(text + p));
            m[0] = newline_mask(v.x) & 0x01010101u; m[1] = newline_mask(v.y) & 0x01010101u;
            m[2] = newline_mask(v.z) & 0x01010101u; m[3] = newline_mask(v.w) & 0x01010101u;
        }
        const uint32_t cnt = __popc(m[0]) + __popc(m[1]) + __popc(m[2]) + __popc(m[3]);
        uint32_t ex, total;
        BS(tmp).ExclusiveSum(cnt, ex, total);
        __syncthreads();
        unsigned long long o = run + ex;
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            uint32_t mk = m[k];
            while (mk) {
                const uint32_t b = (uint32_t)(__ffs((int)mk) - 1) >> 3;
                line_start[++o] = p + (uint32_t)k * 4 + b + 1;
                mk &= mk - 1;
            }
        }
        run += total;
    }
}

struct ParseArgs {
    const uint8_t* text;
    uint64_t n;                       // text bytes
    const unsigned long long* line_start;
    uint64_t n_lines;
    int unterminated;                 // the last line has no '\n' (and so keeps a trailing '\r', misc str::lines semantics)
    TokTable tb;
    tok::LineRec* recs;
    unsigned long long *s_al, *s_ops, *s_blk;   // [n_lines + 1] scan inputs: aligned?, CIGAR ops, sequence blocks
    TokStatus* st;
};

__device__ __forceinline__ void line_span(const ParseArgs& a, tok::Txt& x, uint64_t i, uint64_t& s, uint64_t& e) {
    s = a.line_start[i];
    if (i + 1 == a.n_lines && a.unterminated) { e = a.n; return; }
    e = a.line_start[i + 1] - 1;
    if (e > s && x.at(e - 1) == '\r') e--;
}

__global__ void __launch_bounds__(TK_LINE_THREADS) k_tok_parse(ParseArgs a) {
    __shared__ uint8_t s_nib[256];
    for (int k = threadIdx.x; k < 256; k += TK_LINE_THREADS) s_nib[k] = a.tb.nibtab[k];
    __syncthreads();
    const uint64_t i = (uint64_t)blockIdx.x * TK_LINE_THREADS + threadIdx.x;
    if (i > a.n_lines) return;
    if (i == a.n_lines) { a.s_al[i] = 0; a.s_ops[i] = 0; a.s_blk[i] = 0; return; }
    tok::Txt x(a.text);
    uint64_t s, e;
    line_span(a, x, i, s, e);
    tok::LineRec r;
    const uint8_t kind = tok::parse_line(x, s, e, a.tb.ct, s_nib, r);
    r.kind = kind;
    a.recs[i] = r;
    const bool al = kind == tok::LK_ALIGNED;
    a.s_al[i] = al ? 1 : 0;
    a.s_ops[i] = al ? r.nops : 0;
    a.s_blk[i] = al ? tok::seq_blocks(r) : 0;
    if (kind == tok::LK_HOST) atomicMin(&a.st->first_bad, (unsigned long long)i);
    if (al && r.need8) a.st->need8 = 1;
}

struct EmitArgs {
    ParseArgs p;
    uint64_t aln_base, ops_base, blk_base;
    DsArrays d;                       // the dataset
    unsigned long long* name_pos;     // [alignments of this file] text offset of the QNAME
    uint32_t* name_len;
};

template <int BITS>
__global__ void __launch_bounds__(TK_LINE_THREADS) k_tok_emit(EmitArgs a) {
    __shared__ uint8_t s_nib[256];
    for (int k = threadIdx.x; k < 256; k += TK_LINE_THREADS) s_nib[k] = a.p.tb.nibtab[k];
    __syncthreads();
    const uint64_t i = (uint64_t)blockIdx.x * TK_LINE_THREADS + threadIdx.x;
    if (i >= a.p.n_lines) return;
    const tok::LineRec r = a.p.recs[i];
    if (r.kind != tok::LK_ALIGNED) return;
    const uint64_t s = a.p.line_start[i];
    const uint64_t la = a.p.s_al[i], A = a.aln_base + la;
    const uint64_t co = a.ops_base + a.p.s_ops[i], bo = a.blk_base + a.p.s_blk[i];
    const bool star = r.flags & PP_FLAG_SEQSTAR;
    a.d.contig[A] = r.contig;
    a.d.ref_start[A] = r.ref_start;
    a.d.seq_off[A] = star ? 0u : (uint32_t)bo;
    a.d.seq_len[A] = (uint16_t)r.slen;
    a.d.cigar_off[A] = (uint32_t)co;
    a.d.n_cigar[A] = (uint16_t)r.nops;
    a.d.nm[A] = r.nm;
    a.d.flags[A] = r.flags;
    a.name_pos[la] = s;
    a.name_len[la] = r.name_len;
    tok::Txt x(a.p.text);
    tok::emit_cigar(x, s, r, a.d.cigar_ops + co);
    if (tok::emit_seq<BITS>(x, s, r, s_nib, a.d.seq_pool + bo * ds_block_bytes(BITS))) a.p.st->need8 = 1;
}

__global__ void __launch_bounds__(TK_LINE_THREADS) k_tok_heads(const uint8_t* __restrict__ text, uint64_t n_al, const unsigned long long* __restrict__ name_pos,
                                                               const uint32_t* __restrict__ name_len, uint32_t* __restrict__ head) {
    const uint64_t a = (uint64_t)blockIdx.x * TK_LINE_THREADS + threadIdx.x;
    if (a >= n_al) return;
    tok::Txt x(text);
    head[a] = tok::group_head(x, a, 0, reinterpret_cast<const uint64_t*>(name_pos), name_len) ? 1u : 0u;
}

__global__ void __launch_bounds__(TK_LINE_THREADS) k_tok_groups(uint64_t n_al, const uint32_t* __restrict__ head, const uint32_t* __restrict__ rs, uint64_t read_base,
                                                                int careful, uint32_t* __restrict__ read_id, uint32_t* seq_off, uint16_t* seq_len, uint8_t* flags,
                                                                TokStatus* st) {
    const uint64_t a = (uint64_t)blockIdx.x * TK_LINE_THREADS + threadIdx.x;
    if (a >= n_al) return;
    read_id[a] = (uint32_t)(read_base + rs[a] - 1);
    if (head[a] && !tok::close_group(a, n_al, head, careful != 0, seq_off, seq_len, flags)) st->group_err = 1;
}

}  // namespace

struct TokFilterBufs;

struct TokState {
    const pp_fasta* fasta = nullptr;
    bool careful = false, active = false;
    int seq_bits = 4;
    uint64_t aln_base = 0, ops_base = 0, blk_base = 0, read_base = 0;   // dataset under construction
    TokTable tb{};
    TokStatus* h_st = nullptr;            // pinned
    unsigned long long* h_tot = nullptr;  // pinned [4]
    TokStatus* d_st = nullptr;
    // file streaming
    uint8_t* pin[TK_READERS][2] = {};
    cudaStream_t rstream[TK_READERS] = {};
    cudaEvent_t rev[TK_READERS][2] = {};
    int readers = 0;                      // threads in use (pp_tok_set_readers, default from the core count)
    int ring = 0;                         // readers whose slots / stream exist
    // text buffers: one being tokenised, one being filled by the background upload of the next file
    DevBuf text[2];
    int next_buf = 0;
    uint64_t expect_total = 0;            // pp_tok_expect: bytes of all the files of this dataset (sizes the arrays once)
    struct Prefetch {
        std::thread th;
        bool active = false;
        std::string path;
        int buf = 0;
        uint64_t n = 0;
        uint8_t last = '\n';
        int rc = PP_OK;                   // PP_OK, PP_ERR_IO, PP_ERR_CUDA
        int cuda_err = 0;
        float ms = 0;
        uint64_t off = 0;                 // first byte of the file that is sent (pp_tok_set_ranges)
        bool strip = false;               // uploaded with QUAL replaced by "*" (polish only: filter reproduces lines verbatim)
        uint64_t sent = 0;                // bytes that crossed PCIe
    } pf;
    bool strip_qual = false;              // pp_tok_set_strip_qual (off by default: measured host-bound, see profiles/README.md)
    uint8_t* h_nl = nullptr;              // pinned '\n'
    DevBuf cub;
    TokFilterBufs* fbufs = nullptr;   // device buffers of the filter text path
    // pp_tok_set_ranges: this context tokenises one byte range of every file (multi-GPU ingestion); marks[f] = the dataset's
    // (alignments, ops, sequence blocks, reads) when file f started, marks.back() = now
    bool ranges_on = false;
    std::vector<uint64_t> range_off, range_len;
    struct Mark { uint64_t aln, ops, blk, reads; };
    std::vector<Mark> marks;
    struct XState;                    // buffers of pp_tok_exchange_finish, kept between calls (no cudaMalloc in the steady state)
    XState* xs = nullptr;
    // pp_tok_set_shard: this context keeps one shard of the assembly
    bool shard_on = false, shard_unknown = false;
    DevBuf shard_map;                 // local_of[c] on the device
    uint32_t shard_n_total = 0;
    std::vector<uint64_t> shard_off;
    std::vector<uint8_t> shard_bases;
};

static void free_filter_bufs(TokFilterBufs* b);
static void free_xstate(TokState* T);

void pp_tok_release(pp_ctx* ctx) {
    TokState* T = ctx->tok;
    if (!T) return;
    if (T->fbufs) { free_filter_bufs(T->fbufs); T->fbufs = nullptr; }
    if (T->pf.active && T->pf.th.joinable()) T->pf.th.join();
    T->text[0].release(); T->text[1].release();
    for (int r = 0; r < TK_READERS; ++r) {
        for (int k = 0; k < 2; ++k) {
            if (T->pin[r][k]) cudaFreeHost(T->pin[r][k]);
            if (T->rev[r][k]) cudaEventDestroy(T->rev[r][k]);
        }
        if (T->rstream[r]) cudaStreamDestroy(T->rstream[r]);
    }
    if (T->h_st) cudaFreeHost(T->h_st);
    if (T->h_nl) cudaFreeHost(T->h_nl);
    if (T->h_tot) cudaFreeHost(T->h_tot);
    if (T->d_st) cudaFree(T->d_st);
    T->cub.release();
    T->shard_map.release();
    free_xstate(T);
    delete T;
    ctx->tok = nullptr;
}

static int tok_state(pp_ctx* ctx, TokState** out) {
    if (!ctx->tok) {
        TokState* T = new TokState();
        ctx->tok = T;
        CK(cudaHostAlloc((void**)&T->h_st, sizeof(TokStatus), cudaHostAllocDefault));
        CK(cudaHostAlloc((void**)&T->h_tot, 4 * sizeof(unsigned long long), cudaHostAllocDefault));
        CK(cudaMalloc((void**)&T->d_st, sizeof(TokStatus)));
        CK(cudaHostAlloc((void**)&T->h_nl, 64, cudaHostAllocDefault));
        T->h_nl[0] = '\n';
    }
    *out = ctx->tok;
    return PP_OK;
}

// Grows a dataset buffer keeping its first `keep` bytes (the alignments of the files tokenised so far).
static int ensure_keep(pp_ctx* ctx, int which, size_t bytes, size_t keep) {
    DevBuf& b = ctx->b[which];
    if (bytes <= b.cap) return PP_OK;
    if (keep == 0) { CK(b.ensure(bytes)); return PP_OK; }
    void* np = nullptr;
    const size_t want = bytes + bytes / 4 + 256;
    CK(cudaMalloc(&np, want));
    cudaError_t e = cudaMemcpyAsync(np, b.p, keep, cudaMemcpyDeviceToDevice, ctx->stream);
    if (e == cudaSuccess) e = cudaStreamSynchronize(ctx->stream);
    if (e != cudaSuccess) { cudaFree(np); CK(e); }
    cudaFree(b.p);
    b.p = np;
    b.cap = want;
    return PP_OK;
}

// The line index of a text on the device (n bytes, zero padded), in two calls.  line_count counts its lines - newlines per 16 KiB tile
// (k_tok_count), their offsets (a scan, in B_TOKLINE), the total read back - and answers PP_TOK_HOST past the limits; line_starts then
// writes line_start[0 .. n_lines] into the caller's buffer (k_tok_index).
struct LineIndex { uint64_t n16, n_tiles, n_lines; const unsigned long long* tile_off; };

static int line_count(pp_ctx* ctx, TokState* T, const uint8_t* text, uint64_t n, bool unterminated, LineIndex* li) {
    cudaStream_t s = ctx->stream;
    li->n16 = (n + 15) & ~15ull;
    li->n_tiles = (li->n16 + TK_TILE - 1) / TK_TILE;
    li->n_lines = 0;
    if (li->n_tiles >= 0x7FFFFFFFull) return PP_TOK_HOST;
    size_t cub_bytes = 0;
    CK(cub::DeviceScan::ExclusiveSum(nullptr, cub_bytes, (unsigned long long*)nullptr, (unsigned long long*)nullptr, (int64_t)std::max<uint64_t>(li->n_tiles + 1, 1)));
    CK(T->cub.ensure(cub_bytes + 256));
    TRY_ALLOC(ctx->b[B_TOKLINE].ensure((li->n_tiles + 2) * 8));
    unsigned long long* tile_cnt = ctx->b[B_TOKLINE].as<unsigned long long>();
    li->tile_off = tile_cnt;
    if (li->n_tiles) {
        CK(cudaMemsetAsync(tile_cnt + li->n_tiles, 0, 8, s));
        k_tok_count<<<(unsigned)li->n_tiles, TK_THREADS, 0, s>>>(text, li->n16, tile_cnt);
        size_t tb = T->cub.cap;
        CK(cub::DeviceScan::ExclusiveSum(T->cub.p, tb, tile_cnt, tile_cnt, (int64_t)(li->n_tiles + 1), s));
        CK(cudaMemcpyAsync(T->h_tot, tile_cnt + li->n_tiles, 8, cudaMemcpyDeviceToHost, s));
        CK(cudaStreamSynchronize(s));
        li->n_lines = T->h_tot[0] + (unterminated ? 1 : 0);
    }
    return li->n_lines >= 0xFFFFFFF0ull ? PP_TOK_HOST : PP_OK;
}

static void line_starts(pp_ctx* ctx, const uint8_t* text, const LineIndex& li, unsigned long long* line_start) {
    k_tok_index<<<(unsigned)li.n_tiles, TK_THREADS, 0, ctx->stream>>>(text, li.n16, li.tile_off, line_start);
}

int pp_ctx_upload_contigs(pp_ctx* ctx, const pp_contigs* c);
int pp_ctx_commit_dataset(pp_ctx* ctx, uint64_t n_aln, uint64_t n_reads, uint64_t n_ops, uint64_t seq_bytes, uint32_t seq_bits);

extern "C" int pp_tok_begin(pp_ctx* ctx, const pp_fasta* fa, int careful, int seq_bits) {
    if (!ctx) return PP_ERR_ARG;
    if (!fa || (seq_bits != 4 && seq_bits != 8)) return ctx->fail(PP_ERR_ARG, "pp_tok_begin: null assembly or seq_bits not 4 / 8");
    CK(cudaSetDevice(ctx->device));
    TokState* T = nullptr;
    int rc = tok_state(ctx, &T);
    if (rc) return rc;
    ctx->have_ds = false;
    pp_contigs contigs;
    pp_fasta_view(fa, &contigs);
    if ((rc = pp_ctx_upload_contigs(ctx, &contigs))) return rc;
    tok::TableImage im;
    tok::build_table_image(fa->names, im);
    CK(ctx->b[B_TOKNAMES].ensure(im.bytes.size()));
    CK(cudaMemcpyAsync(ctx->b[B_TOKNAMES].p, im.bytes.data(), im.bytes.size(), cudaMemcpyHostToDevice, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));              // `im` is pageable and about to go away
    const uint8_t* base = ctx->b[B_TOKNAMES].as<uint8_t>();
    T->tb.ct = tok::table_view(im, base);
    T->tb.nibtab = base + im.o_nib;
    T->fasta = fa; T->careful = careful != 0; T->seq_bits = seq_bits;
    T->aln_base = T->ops_base = T->blk_base = T->read_base = 0;
    T->expect_total = 0;
    T->active = true;
    T->shard_on = false;
    T->ranges_on = false;
    T->marks.clear();
    return PP_OK;
}

// Optional, after pp_tok_begin: the i-th path of pp_tok_add_files contributes only bytes [off[i], off[i] + len[i]) - a range that
// starts at a line start and ends behind a line end, cut between two read groups (the caller's job: host_api.cpp split_ranges).
// A range without alignments is fine (the file as a whole is the caller's to check).
extern "C" int pp_tok_set_ranges(pp_ctx* ctx, const uint64_t* off, const uint64_t* len, int n) {
    if (!ctx) return PP_ERR_ARG;
    TokState* T = ctx->tok;
    if (!T || !T->active) return ctx->fail(PP_ERR_ARG, "pp_tok_set_ranges: no pp_tok_begin");
    if (n < 0 || (n && (!off || !len))) return ctx->fail(PP_ERR_ARG, "pp_tok_set_ranges: null ranges");
    T->range_off.assign(off, off + n);
    T->range_len.assign(len, len + n);
    T->ranges_on = true;
    return PP_OK;
}

// Records of contigs this shard does not hold become ghosts (shard.cpp does the same on the host: contig 0, PP_FLAG_GHOST); the rest
// get the shard's contig numbers.
__global__ void k_shard_mark(uint32_t* __restrict__ contig, uint8_t* __restrict__ flags, uint64_t n_aln, const uint32_t* __restrict__ local_of,
                             uint32_t n_total, int takes_unknown) {
    for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < n_aln; i += (uint64_t)gridDim.x * blockDim.x) {
        const uint32_t c = contig[i];
        uint32_t l = 0xFFFFFFFFu;
        if (c == PP_CONTIG_UNKNOWN || c >= n_total) { if (takes_unknown) continue; }
        else l = local_of[c];
        if (l == 0xFFFFFFFFu) { contig[i] = 0; flags[i] |= PP_FLAG_GHOST; }
        else contig[i] = l;
    }
}

extern "C" int pp_tok_set_shard(pp_ctx* ctx, const uint32_t* local_of, uint32_t n_contigs_total, const pp_contigs* sc, int takes_unknown) {
    if (!ctx) return PP_ERR_ARG;
    TokState* T = ctx->tok;
    if (!T || !T->active) return ctx->fail(PP_ERR_ARG, "pp_tok_set_shard: no pp_tok_begin");
    if (!local_of || !sc || !sc->off || !sc->bases || sc->n_contigs == 0) return ctx->fail(PP_ERR_ARG, "pp_tok_set_shard: null or empty shard");
    for (uint32_t c = 0; c < n_contigs_total; ++c)
        if (local_of[c] != 0xFFFFFFFFu && local_of[c] >= sc->n_contigs) return ctx->fail(PP_ERR_ARG, "pp_tok_set_shard: local index outside the shard");
    CK(cudaSetDevice(ctx->device));
    CK(T->shard_map.ensure((size_t)n_contigs_total * 4 + 16));
    CK(cudaMemcpyAsync(T->shard_map.p, local_of, (size_t)n_contigs_total * 4, cudaMemcpyHostToDevice, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    T->shard_off.assign(sc->off, sc->off + sc->n_contigs + 1);
    T->shard_bases.assign(sc->bases, sc->bases + sc->off[sc->n_contigs]);
    T->shard_n_total = n_contigs_total;
    T->shard_unknown = takes_unknown != 0;
    T->shard_on = true;
    return PP_OK;
}

// The text is on the device (n bytes, zero padded).  Appends its alignments to the dataset under construction.
static int tok_process(pp_ctx* ctx, TokState* T, const uint8_t* text, uint64_t n, bool unterminated, pp_tok_stats* stats, bool part_of_file = false) {
    cudaStream_t s = ctx->stream;
    uint32_t launches = 0;
    CK(cudaEventRecord(ctx->ev[0], s));
    // ---- lines
    LineIndex li;
    int rc = line_count(ctx, T, text, n, unterminated, &li);
    const uint64_t n_lines = li.n_lines;
    if (stats) stats->lines = n_lines;
    if (rc != PP_OK) return rc;
    if (li.n_tiles) launches += 3;
    if (n_lines == 0) return part_of_file ? PP_OK : PP_TOK_HOST;   // "no alignments in <file>": the host packer words it (a byte range may be empty)

    // scratch: line starts | line records | three scan arrays
    size_t off = 0;
    auto carve = [&](size_t bytes) { size_t o = off; off += (bytes + 255) & ~size_t(255); return o; };
    const size_t o_ls = carve((n_lines + 2) * 8), o_rec = carve(n_lines * sizeof(tok::LineRec)), o_al = carve((n_lines + 1) * 8),
                 o_ops = carve((n_lines + 1) * 8), o_blk = carve((n_lines + 1) * 8);
    TRY_ALLOC(ctx->b[B_TOKTMP].ensure(off));
    uint8_t* tmp = ctx->b[B_TOKTMP].as<uint8_t>();
    ParseArgs pa;
    pa.text = text; pa.n = n; pa.line_start = (unsigned long long*)(tmp + o_ls); pa.n_lines = n_lines; pa.unterminated = unterminated ? 1 : 0;
    pa.tb = T->tb; pa.recs = (tok::LineRec*)(tmp + o_rec);
    pa.s_al = (unsigned long long*)(tmp + o_al); pa.s_ops = (unsigned long long*)(tmp + o_ops); pa.s_blk = (unsigned long long*)(tmp + o_blk);
    pa.st = T->d_st;
    T->h_st->first_bad = ~0ull; T->h_st->need8 = 0; T->h_st->group_err = 0;
    CK(cudaMemcpyAsync(T->d_st, T->h_st, sizeof(TokStatus), cudaMemcpyHostToDevice, s));
    line_starts(ctx, text, li, (unsigned long long*)(tmp + o_ls));
    const unsigned line_grid = (unsigned)((n_lines + 1 + TK_LINE_THREADS - 1) / TK_LINE_THREADS);
    k_tok_parse<<<line_grid, TK_LINE_THREADS, 0, s>>>(pa);
    size_t cub_bytes = 0;
    CK(cub::DeviceScan::ExclusiveSum(nullptr, cub_bytes, pa.s_al, pa.s_al, (int64_t)(n_lines + 1)));
    CK(T->cub.ensure(cub_bytes + 256));
    for (unsigned long long* arr : {pa.s_al, pa.s_ops, pa.s_blk}) {
        size_t tb = T->cub.cap;
        CK(cub::DeviceScan::ExclusiveSum(T->cub.p, tb, arr, arr, (int64_t)(n_lines + 1), s));
    }
    CK(cudaMemcpyAsync(T->h_tot + 0, pa.s_al + n_lines, 8, cudaMemcpyDeviceToHost, s));
    CK(cudaMemcpyAsync(T->h_tot + 1, pa.s_ops + n_lines, 8, cudaMemcpyDeviceToHost, s));
    CK(cudaMemcpyAsync(T->h_tot + 2, pa.s_blk + n_lines, 8, cudaMemcpyDeviceToHost, s));
    CK(cudaMemcpyAsync(T->h_st, T->d_st, sizeof(TokStatus), cudaMemcpyDeviceToHost, s));
    CK(cudaStreamSynchronize(s));
    launches += 5;
    const uint64_t n_al = T->h_tot[0], n_ops = T->h_tot[1], n_blk = T->h_tot[2];
    if (stats) stats->alignments = n_al;
    if (T->h_st->first_bad != ~0ull) return PP_TOK_HOST;
    if (n_al == 0) return part_of_file ? PP_OK : PP_TOK_HOST;      // alignment.rs:268-270
    if (T->aln_base + n_al >= 0xFFFFFFFFull - 4096 || T->ops_base + n_ops > 0xFFFFFFFFull || T->blk_base + n_blk > 0xFFFFFFFFull) return PP_TOK_HOST;

    // ---- dataset arrays (kept across files)
    const uint64_t A0 = T->aln_base, A1 = A0 + n_al;
    // first file of a dataset whose total text size is known: size the arrays for all of it (no regrowth, no cudaFree later)
    double grow = 1.0;
    if (A0 == 0 && T->expect_total > n && n > 0) grow = std::min(64.0, 1.03 * (double)T->expect_total / (double)n);
    auto want = [&](uint64_t items, size_t each) { return (size_t)((double)items * grow) * each; };
    const uint64_t have[3] = {A0, T->ops_base, T->blk_base}, add[3] = {n_al, n_ops, n_blk};
    for (int k = 0; k < DS_N; ++k) {
        const uint64_t h = have[DS_ARRAYS[k].count], a = add[DS_ARRAYS[k].count];
        const size_t w = ds_width(k, T->seq_bits), pad = k == DS_SEQPOOL ? 256 : 64;
        if ((rc = ensure_keep(ctx, B_CONTIG + k, std::max<size_t>((h + a) * w, want(a, w)) + pad, h * w))) return rc;
    }
    // per-alignment scratch of this file: QNAME position / length, group heads, their running count
    size_t off2 = 0;
    auto carve2 = [&](size_t bytes) { size_t o = off2; off2 += (bytes + 255) & ~size_t(255); return o; };
    const size_t o_np = carve2(n_al * 8), o_nl = carve2(n_al * 4), o_hd = carve2(n_al * 4), o_rs = carve2(n_al * 4);
    TRY_ALLOC(ctx->b[B_SCRATCH].ensure(off2));
    uint8_t* sc = ctx->b[B_SCRATCH].as<uint8_t>();

    EmitArgs ea;
    ea.p = pa; ea.aln_base = A0; ea.ops_base = T->ops_base; ea.blk_base = T->blk_base;
    ea.d = ds_view(ctx->b + B_CONTIG);
    ea.name_pos = (unsigned long long*)(sc + o_np); ea.name_len = (uint32_t*)(sc + o_nl);
    const unsigned emit_grid = (unsigned)((n_lines + TK_LINE_THREADS - 1) / TK_LINE_THREADS);
    if (T->seq_bits == 4) k_tok_emit<4><<<emit_grid, TK_LINE_THREADS, 0, s>>>(ea);
    else k_tok_emit<8><<<emit_grid, TK_LINE_THREADS, 0, s>>>(ea);
    uint32_t* head = (uint32_t*)(sc + o_hd);
    uint32_t* rs = (uint32_t*)(sc + o_rs);
    const unsigned aln_grid = (unsigned)((n_al + TK_LINE_THREADS - 1) / TK_LINE_THREADS);
    k_tok_heads<<<aln_grid, TK_LINE_THREADS, 0, s>>>(text, n_al, ea.name_pos, ea.name_len, head);
    CK(cub::DeviceScan::InclusiveSum(nullptr, cub_bytes, head, rs, (int64_t)n_al));
    CK(T->cub.ensure(cub_bytes + 256));
    {
        size_t tb = T->cub.cap;
        CK(cub::DeviceScan::InclusiveSum(T->cub.p, tb, head, rs, (int64_t)n_al, s));
    }
    k_tok_groups<<<aln_grid, TK_LINE_THREADS, 0, s>>>(n_al, head, rs, T->read_base, T->careful ? 1 : 0, ea.d.read_id + A0,
                                                       ea.d.seq_off + A0, ea.d.seq_len + A0, ea.d.flags + A0, T->d_st);
    uint32_t* h_reads = (uint32_t*)(T->h_tot + 3);
    CK(cudaMemcpyAsync(h_reads, rs + (n_al - 1), 4, cudaMemcpyDeviceToHost, s));
    CK(cudaMemcpyAsync(T->h_st, T->d_st, sizeof(TokStatus), cudaMemcpyDeviceToHost, s));
    CK(cudaEventRecord(ctx->ev[1], s));
    CK(cudaStreamSynchronize(s));
    CK(cudaGetLastError());
    launches += 4;
    if (T->h_st->group_err) return PP_TOK_HOST;
    if (T->h_st->need8 && T->seq_bits == 4) return PP_TOK_NEED8;   // found while the bases were converted (k_tok_emit)
    const uint64_t n_reads = *h_reads;
    if (T->read_base + n_reads >= 0xFFFFFFFFull) return PP_TOK_HOST;
    T->aln_base = A1; T->ops_base += n_ops; T->blk_base += n_blk; T->read_base += n_reads;
    if (stats) {
        stats->reads = n_reads;
        float ms = 0;
        CK(cudaEventElapsedTime(&ms, ctx->ev[0], ctx->ev[1]));
        stats->device_ms = ms;
        stats->launches = launches;
    }
    return PP_OK;
}

static int text_buffer(pp_ctx* ctx, DevBuf& tb, uint64_t n) {
    CK(tb.ensure(n + 64));
    const uint64_t n16 = (n + 15) & ~15ull;
    CK(cudaMemsetAsync(tb.as<uint8_t>() + n, 0, (size_t)(n16 + 32 - n), ctx->stream));   // the copies never touch [n, ...)
    return PP_OK;
}

extern "C" int pp_tok_add_text(pp_ctx* ctx, const char* text, size_t len, pp_tok_stats* stats) {
    if (!ctx) return PP_ERR_ARG;
    TokState* T = ctx->tok;
    if (!T || !T->active) return ctx->fail(PP_ERR_ARG, "pp_tok_add_text: no pp_tok_begin");
    if (!text && len) return ctx->fail(PP_ERR_ARG, "pp_tok_add_text: null text");
    CK(cudaSetDevice(ctx->device));
    if (stats) memset(stats, 0, sizeof *stats);
    if (T->pf.active) { if (T->pf.th.joinable()) T->pf.th.join(); T->pf.active = false; }
    DevBuf& tb = T->text[T->next_buf];
    T->next_buf ^= 1;
    int rc = text_buffer(ctx, tb, len);
    if (rc) return rc;
    const auto t0 = std::chrono::steady_clock::now();
    if (len) CK(cudaMemcpyAsync(tb.p, text, len, cudaMemcpyHostToDevice, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    const float h2d = std::chrono::duration<float, std::milli>(std::chrono::steady_clock::now() - t0).count();
    rc = tok_process(ctx, T, tb.as<uint8_t>(), len, len > 0 && text[len - 1] != '\n', stats);
    if (stats) { stats->h2d_ms = h2d; stats->h2d_bytes = len; }
    if (rc != PP_OK) T->active = false;
    return rc;
}

// Streams a file into dst: T->readers host threads, each pread()s its slices into its two pinned slots and sends them on
// its own stream, so that page-cache reads, pinned staging and PCIe overlap.  Runs on the caller's thread or on the
// prefetch thread; touches neither ctx->err nor ctx->stream.  Returns PP_OK / PP_ERR_IO / PP_ERR_CUDA (+ *cuda_err).
static int upload_file(int device, TokState* T, uint8_t* dst, int fd, uint64_t n, uint8_t* last_byte, int* cuda_err, uint64_t foff = 0) {
    const int R = T->readers;
    const uint64_t n_slices = (n + TK_SLOT - 1) / TK_SLOT;
    std::atomic<int> err{0};           // 1 = read error, 2 = CUDA error
    std::atomic<int> cerr{0};
    auto work = [&](int r) {
        if (cudaSetDevice(device) != cudaSuccess) { err = 2; return; }
        uint64_t k = 0;
        for (uint64_t sl = (uint64_t)r; sl < n_slices && !err; sl += (uint64_t)R, ++k) {
            const int slot = (int)(k & 1);
            if (k >= 2) {
                cudaError_t e = cudaEventSynchronize(T->rev[r][slot]);
                if (e != cudaSuccess) { cerr = (int)e; err = 2; return; }
            }
            const uint64_t o = sl * TK_SLOT, len = std::min<uint64_t>(TK_SLOT, n - o);
            uint64_t got = 0;
            while (got < len) {
                const ssize_t g = pread(fd, T->pin[r][slot] + got, (size_t)(len - got), (off_t)(foff + o + got));
                if (g <= 0) { err = 1; return; }
                got += (uint64_t)g;
            }
            if (o + len == n) *last_byte = T->pin[r][slot][len - 1];
            cudaError_t e = cudaMemcpyAsync(dst + o, T->pin[r][slot], (size_t)len, cudaMemcpyHostToDevice, T->rstream[r]);
            if (e == cudaSuccess) e = cudaEventRecord(T->rev[r][slot], T->rstream[r]);
            if (e != cudaSuccess) { cerr = (int)e; err = 2; return; }
        }
        cudaError_t e = cudaStreamSynchronize(T->rstream[r]);
        if (e != cudaSuccess) { cerr = (int)e; err = 2; }
    };
    std::vector<std::thread> th;
    for (int r = 1; r < R; ++r) th.emplace_back(work, r);
    work(0);
    for (auto& t : th) t.join();
    *cuda_err = cerr.load();
    return err == 1 ? PP_ERR_IO : err == 2 ? PP_ERR_CUDA : PP_OK;
}

constexpr int PP_UPLOAD_LONG_LINE = 100;   // internal: a line longer than TK_LOOK, upload the file verbatim instead

// The same for `polish`, with less on the wire: every reader owns the LINES that start in its nominal slice, replaces their
// QUAL by "*" while staging them (tok_strip.h: 45 % of a bwa-mem line, never read on this path) and sends the shorter text
// to the lines' original offset; the freed tail of the slice becomes one '@' comment line on the device ('@', blanks
// written by a memset, '\n'), which every parser of this path skips (alignment.rs:241-242).  Offsets, and therefore the
// independence of the readers, stay as they are.  A file whose last line is unterminated keeps its last slice verbatim.
static int upload_file_stripped(int device, TokState* T, uint8_t* dst, int fd, uint64_t n, uint8_t* last_byte, int* cuda_err, uint64_t* sent) {
    const int R = T->readers;
    const uint64_t S = TK_SLOT - TK_LOOK;
    const uint64_t n_slices = (n + S - 1) / S;
    std::atomic<int> err{0}, cerr{0};              // 1 read error, 2 CUDA error, 3 long line
    std::atomic<unsigned long long> bytes{0};
    // the lines are read through a private mapping of the file where that works (no copy before the strip), else pread
    const uint8_t* map = nullptr;
    {
        void* m = n ? mmap(nullptr, (size_t)n, PROT_READ, MAP_PRIVATE, fd, 0) : MAP_FAILED;
        if (m != MAP_FAILED) { map = (const uint8_t*)m; madvise(m, (size_t)n, MADV_SEQUENTIAL); }
    }
    auto work = [&](int r) {
        if (cudaSetDevice(device) != cudaSuccess) { err = 2; return; }
        std::vector<uint8_t> rawbuf(map ? 16 : TK_SLOT + 16);
        uint64_t j = 0;
        for (uint64_t k = (uint64_t)r; k < n_slices && !err; k += (uint64_t)R) {
            const uint64_t o = k * S, e = std::min<uint64_t>(n, o + S);
            const uint64_t rd0 = k ? o - 1 : 0, rd1 = std::min<uint64_t>(n, e + TK_LOOK - 1);
            const uint8_t* raw = map ? map + rd0 : rawbuf.data();
            if (!map) {
                uint64_t got = 0;
                while (got < rd1 - rd0) {
                    const ssize_t g = pread(fd, rawbuf.data() + got, (size_t)(rd1 - rd0 - got), (off_t)(rd0 + got));
                    if (g <= 0) { err = 1; return; }
                    got += (uint64_t)g;
                }
            }
            // the slot is needed before the lines are staged into it
            const int slot = (int)(j & 1);
            if (j >= 2) {
                cudaError_t ce = cudaEventSynchronize(T->rev[r][slot]);
                if (ce != cudaSuccess) { cerr = (int)ce; err = 2; return; }
            }
            uint8_t* pin = T->pin[r][slot];
            const tok::SliceOut so = tok::strip_slice(raw, rd0, rd1, k, e, n, pin);
            if (so.status == 3) { err = 3; return; }
            if (so.status == 1) continue;                          // one long line covers the whole slice: an earlier slice owns it
            ++j;
            if (so.ends_file) *last_byte = so.last;
            const uint64_t a = so.a, b = so.b, c = so.c, gap = (b - a) - c;
            cudaError_t ce = cudaSuccess;
            if (gap == 0) {
                ce = cudaMemcpyAsync(dst + a, pin, (size_t)c, cudaMemcpyHostToDevice, T->rstream[r]);
            } else if (gap == 1) {
                pin[c] = '\n';                                      // an empty line
                ce = cudaMemcpyAsync(dst + a, pin, (size_t)c + 1, cudaMemcpyHostToDevice, T->rstream[r]);
            } else {
                pin[c] = '@';                                       // a comment line of gap bytes
                ce = cudaMemcpyAsync(dst + a, pin, (size_t)c + 1, cudaMemcpyHostToDevice, T->rstream[r]);
                if (ce == cudaSuccess && gap > 2) ce = cudaMemsetAsync(dst + a + c + 1, ' ', (size_t)(gap - 2), T->rstream[r]);
                if (ce == cudaSuccess) ce = cudaMemcpyAsync(dst + b - 1, T->h_nl, 1, cudaMemcpyHostToDevice, T->rstream[r]);
            }
            if (ce == cudaSuccess) ce = cudaEventRecord(T->rev[r][slot], T->rstream[r]);
            if (ce != cudaSuccess) { cerr = (int)ce; err = 2; return; }
            bytes += c + (gap ? 2 : 0);
        }
        cudaError_t ce = cudaStreamSynchronize(T->rstream[r]);
        if (ce != cudaSuccess) { cerr = (int)ce; err = 2; }
    };
    std::vector<std::thread> th;
    for (int r = 1; r < R; ++r) th.emplace_back(work, r);
    work(0);
    for (auto& t : th) t.join();
    if (map) munmap((void*)map, (size_t)n);
    *cuda_err = cerr.load();
    *sent = bytes.load();
    if (err == 3) {                                   // let the copies that were issued finish before the verbatim upload reuses the slots
        for (int r = 0; r < R; ++r) cudaStreamSynchronize(T->rstream[r]);
        return PP_UPLOAD_LONG_LINE;
    }
    return err == 1 ? PP_ERR_IO : err == 2 ? PP_ERR_CUDA : PP_OK;
}

static int ring_ready(pp_ctx* ctx, TokState* T) {
    if (T->readers <= 0) {
        const unsigned hw = std::thread::hardware_concurrency();
        T->readers = (int)std::min<unsigned>(TK_READERS, std::max<unsigned>(2, hw / 4));
    }
    for (int r = T->ring; r < T->readers; ++r) {
        CK(cudaStreamCreateWithFlags(&T->rstream[r], cudaStreamNonBlocking));
        for (int k = 0; k < 2; ++k) {
            CK(cudaHostAlloc((void**)&T->pin[r][k], TK_SLOT, cudaHostAllocDefault));
            CK(cudaEventCreateWithFlags(&T->rev[r][k], cudaEventDisableTiming));
        }
        T->ring = r + 1;
    }
    return PP_OK;
}

// Starts streaming `path` into the next text buffer on a background thread.  PP_OK, PP_TOK_HOST (not a plain readable
// file) or an error.
static int prefetch_start(pp_ctx* ctx, TokState* T, const char* path, bool strip, int range = -1) {
    struct stat sb;
    if (stat(path, &sb) != 0 || !S_ISREG(sb.st_mode)) return PP_TOK_HOST;   // pipes, devices: never opened here (the host path streams them once)
    const int fd = open(path, O_RDONLY);
    if (fd < 0 || fstat(fd, &sb) != 0 || !S_ISREG(sb.st_mode)) {
        if (fd >= 0) close(fd);
        return PP_TOK_HOST;
    }
    uint64_t n = (uint64_t)sb.st_size, foff = 0;
    if (range >= 0) {
        if ((size_t)range >= T->range_off.size() || T->range_off[range] + T->range_len[range] > n) { close(fd); return PP_TOK_HOST; }
        foff = T->range_off[range]; n = T->range_len[range];
        strip = false;                                           // (the stripping upload works on whole files)
    }
    const int buf = T->next_buf;
    int rc = ring_ready(ctx, T);
    if (rc != PP_OK) { close(fd); return rc; }
    if (T->text[buf].cap < n + 64) {
        // The text, its line index / records and the arrays built from it must fit beside what is already resident; a file too
        // large for that goes through the host parser (which needs no device memory for text).
        size_t free_b = 0, total_b = 0;
        if (cudaMemGetInfo(&free_b, &total_b) != cudaSuccess || (double)free_b + (double)T->text[buf].cap < 2.6 * (double)n + (256 << 20)) {
            cudaGetLastError();
            close(fd);
            return PP_TOK_HOST;
        }
    }
    rc = text_buffer(ctx, T->text[buf], n);
    if (rc != PP_OK) { cudaGetLastError(); close(fd); return PP_TOK_HOST; }
    T->next_buf ^= 1;
    TokState::Prefetch& pf = T->pf;
    pf.active = true; pf.path = path; pf.buf = buf; pf.n = n; pf.last = '\n'; pf.rc = PP_OK; pf.cuda_err = 0; pf.ms = 0;
    pf.strip = strip && T->strip_qual; pf.sent = 0; pf.off = foff;
    uint8_t* dst = T->text[buf].as<uint8_t>();
    const int device = ctx->device;
    pf.th = std::thread([T, dst, fd, n, device, foff] {
        TokState::Prefetch& q = T->pf;
        const auto t0 = std::chrono::steady_clock::now();
        if (n && q.strip) {
            q.rc = upload_file_stripped(device, T, dst, fd, n, &q.last, &q.cuda_err, &q.sent);
            if (q.rc == PP_UPLOAD_LONG_LINE) q.strip = false;
        }
        if (n && !q.strip) { q.rc = upload_file(device, T, dst, fd, n, &q.last, &q.cuda_err, foff); q.sent = n; }
        close(fd);
        q.ms = std::chrono::duration<float, std::milli>(std::chrono::steady_clock::now() - t0).count();
    });
    return PP_OK;
}

// Waits for the text of `path` (starting its upload now if nobody asked for it before).
static int prefetch_wait(pp_ctx* ctx, TokState* T, const char* path, bool strip, int range = -1) {
    TokState::Prefetch& pf = T->pf;
    const bool other_range = range >= 0 && (size_t)range < T->range_off.size() && (pf.off != T->range_off[range] || pf.n != T->range_len[range]);
    if (pf.active && (pf.path != path || (pf.strip && !strip) || other_range || (range < 0 && pf.off != 0))) {   // (text without QUAL is no use to `filter`)                       // something else was prefetched: let it finish, drop it
        if (pf.th.joinable()) pf.th.join();
        pf.active = false;
    }
    if (!pf.active) {
        const int rc = prefetch_start(ctx, T, path, strip, range);
        if (rc != PP_OK) return rc;
    }
    if (pf.th.joinable()) pf.th.join();
    pf.active = false;
    if (pf.rc == PP_ERR_IO) return PP_TOK_HOST;               // the host path reports unreadable files
    if (pf.rc == PP_ERR_CUDA) return ctx->fail_cuda((cudaError_t)pf.cuda_err, "SAM text upload", __FILE__, __LINE__);
    return PP_OK;
}

extern "C" int pp_tok_prefetch(pp_ctx* ctx, const char* path) {
    if (!ctx || !path) return PP_ERR_ARG;
    CK(cudaSetDevice(ctx->device));
    TokState* T = nullptr;
    int rc = tok_state(ctx, &T);
    if (rc) return rc;
    if (T->pf.active) return PP_OK;                            // one outstanding upload at a time
    rc = prefetch_start(ctx, T, path, true);
    return rc == PP_TOK_HOST ? PP_OK : rc;                     // pp_tok_add_file(s) will say so
}

extern "C" int pp_tok_expect(pp_ctx* ctx, uint64_t total_text_bytes) {
    if (!ctx) return PP_ERR_ARG;
    TokState* T = nullptr;
    int rc = tok_state(ctx, &T);
    if (rc) return rc;
    T->expect_total = total_text_bytes;
    return PP_OK;
}

extern "C" int pp_tok_add_files(pp_ctx* ctx, const char* const* paths, int n_paths, pp_tok_stats* stats) {
    if (!ctx) return PP_ERR_ARG;
    TokState* T = ctx->tok;
    if (!T || !T->active) return ctx->fail(PP_ERR_ARG, "pp_tok_add_file: no pp_tok_begin");
    if (!paths || n_paths < 0) return ctx->fail(PP_ERR_ARG, "pp_tok_add_file: null paths");
    CK(cudaSetDevice(ctx->device));
    if (stats) memset(stats, 0, sizeof(pp_tok_stats) * (size_t)n_paths);
    if (T->ranges_on && T->range_off.size() != (size_t)n_paths) return ctx->fail(PP_ERR_ARG, "pp_tok_add_files: as many paths as pp_tok_set_ranges ranges");
    const bool ranges = T->ranges_on;
    for (int i = 0; i < n_paths; ++i) {
        if (!paths[i]) return ctx->fail(PP_ERR_ARG, "pp_tok_add_file: null path");
        T->marks.push_back({T->aln_base, T->ops_base, T->blk_base, T->read_base});
        int rc = prefetch_wait(ctx, T, paths[i], true, ranges ? i : -1);
        if (rc != PP_OK) { T->active = false; return rc; }
        const int buf = T->pf.buf;
        const uint64_t n = T->pf.n;
        const bool unterminated = n > 0 && T->pf.last != '\n';
        const float h2d = T->pf.ms;
        const uint64_t h2d_bytes = T->pf.sent;
        if (i + 1 < n_paths && paths[i + 1]) {                 // the next file streams in while this one is tokenised
            rc = prefetch_start(ctx, T, paths[i + 1], true, ranges ? i + 1 : -1);
            if (rc < 0) { T->active = false; return rc; }
        }
        rc = tok_process(ctx, T, T->text[buf].as<uint8_t>(), n, unterminated, stats ? stats + i : nullptr, ranges);
        if (stats) { stats[i].h2d_ms = h2d; stats[i].h2d_bytes = h2d_bytes; }
        if (rc != PP_OK) { T->active = false; return rc; }
    }
    T->marks.push_back({T->aln_base, T->ops_base, T->blk_base, T->read_base});
    return PP_OK;
}

extern "C" int pp_tok_add_file(pp_ctx* ctx, const char* path, pp_tok_stats* stats) {
    return pp_tok_add_files(ctx, &path, 1, stats);
}

extern "C" int pp_set_parser(pp_ctx* ctx, int mode) {
    if (!ctx || mode < 0 || mode > 1) return PP_ERR_ARG;
    ctx->parser = mode;
    return PP_OK;
}
extern "C" int pp_get_parser(const pp_ctx* ctx) { return ctx ? ctx->parser : 0; }

// Host threads that stream a SAM file into the device (0 = from the core count: a quarter of them, 2..16).
extern "C" int pp_tok_set_readers(pp_ctx* ctx, int n) {
    if (!ctx || n < 0 || n > TK_READERS) return PP_ERR_ARG;
    TokState* T = nullptr;
    int rc = tok_state(ctx, &T);
    if (rc) return rc;
    T->readers = n;
    return PP_OK;
}

// 1: pp_tok_add_file(s) / pp_tok_prefetch send the text without its QUAL column; 0 (default): byte for byte.
extern "C" int pp_tok_set_strip_qual(pp_ctx* ctx, int on) {
    if (!ctx) return PP_ERR_ARG;
    TokState* T = nullptr;
    int rc = tok_state(ctx, &T);
    if (rc) return rc;
    T->strip_qual = on != 0;
    return PP_OK;
}

extern "C" int pp_tok_finish(pp_ctx* ctx) {
    if (!ctx) return PP_ERR_ARG;
    TokState* T = ctx->tok;
    if (!T || !T->active) return ctx->fail(PP_ERR_ARG, "pp_tok_finish: no tokenised text");
    T->active = false;
    if (T->shard_on) {
        T->shard_on = false;
        CK(cudaSetDevice(ctx->device));
        if (T->aln_base)
            k_shard_mark<<<(uint32_t)std::min<uint64_t>((T->aln_base + 255) / 256, (uint64_t)ctx->sm_count * 32), 256, 0, ctx->stream>>>(
                ctx->b[B_CONTIG].as<uint32_t>(), ctx->b[B_FLAGS].as<uint8_t>(), T->aln_base, T->shard_map.as<uint32_t>(), T->shard_n_total,
                T->shard_unknown ? 1 : 0);
        pp_contigs sc;
        sc.n_contigs = (uint32_t)T->shard_off.size() - 1; sc.off = T->shard_off.data(); sc.bases = T->shard_bases.data();
        int rc = pp_ctx_upload_contigs(ctx, &sc);           // the shard's contigs are the draft from here on
        if (rc != PP_OK) return rc;
        CK(cudaStreamSynchronize(ctx->stream));             // (pageable sources)
        CK(cudaGetLastError());
        std::vector<uint8_t>().swap(T->shard_bases);
    }
    return pp_ctx_commit_dataset(ctx, T->aln_base, T->read_base, T->ops_base, T->blk_base * ds_block_bytes(T->seq_bits), (uint32_t)T->seq_bits);
}

// fn(side, g) on every context S[g].ctx, each on its own host thread but the first, which runs on the calling thread; the first error
// (its message moved to S[0]'s context) before PP_TOK_HOST, before PP_TOK_NEED8.
template <class Side, class F>
static int fx_all(std::vector<Side>& S, F&& fn) {
    std::vector<int> rc(S.size(), PP_OK);
    auto run = [&](size_t g) {
        pp_ctx* ctx = S[g].ctx;
        const cudaError_t e = cudaSetDevice(ctx->device);
        rc[g] = e != cudaSuccess ? ctx->fail_cuda(e, "cudaSetDevice", __FILE__, __LINE__) : fn(S[g], (int)g);
    };
    std::vector<std::thread> th;
    for (size_t g = 1; g < S.size(); ++g) th.emplace_back(run, g);
    run(0);
    for (auto& t : th) t.join();
    for (size_t g = 0; g < S.size(); ++g)
        if (rc[g] < 0) { if (g) S[0].ctx->err = S[g].ctx->err; return rc[g]; }
    for (int want : {PP_TOK_HOST, PP_TOK_NEED8})
        if (std::count(rc.begin(), rc.end(), want)) return want;
    return PP_OK;
}

// A device-to-device copy on ctx's stream into dctx's memory: a peer copy between two devices.
static int fx_copy(pp_ctx* ctx, pp_ctx* dctx, void* dst, const void* src, size_t bytes) {
    if (!bytes) return PP_OK;
    if (dctx->device == ctx->device) CK(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToDevice, ctx->stream));
    else CK(cudaMemcpyPeerAsync(dst, dctx->device, src, ctx->device, bytes, ctx->stream));
    return PP_OK;
}

// Peer access from ctx's device to the other devices of ctxs: NVLink between the GPUs where the box has it.
static void enable_peers(pp_ctx* ctx, pp_ctx* const* ctxs, size_t n) {
    for (size_t o = 0; o < n; ++o)
        if (ctxs[o]->device != ctx->device) {
            int can = 0;
            if (cudaDeviceCanAccessPeer(&can, ctx->device, ctxs[o]->device) == cudaSuccess && can) cudaDeviceEnablePeerAccess(ctxs[o]->device, 0);
            cudaGetLastError();                                                        // (already enabled is fine)
        }
}

// =====================================================================================================================
// Multi-GPU ingestion without the host in the middle (SURVEY.md §8e at file level).  Every context has tokenised ITS byte range of
// every SAM file (pp_tok_set_ranges; the ranges are cut between read groups).  pp_tok_exchange_finish then gives every GPU its
// shard: a read group goes - whole, so that k still spans contigs - to every GPU that owns a contig one of its records lies on.
// Per source GPU g and destination o: a bit mask per group (k_x_touch), four exclusive scans over the kept records (records, CIGAR
// ops, sequence blocks, groups), a compaction into staging arrays with every offset already renumbered for its place in o's
// dataset (k_x_pack*), and device-to-device copies (cudaMemcpyPeerAsync, NVLink where the box has it) into o's arrays at
// [file f][range g] - global SAM order is (file, range, line), which is what the ordered depth needs.  The host only adds up
// the piece sizes.  Then pp_tok_set_shard / pp_tok_finish on every GPU: foreign records become ghosts, the shard is binned.
// =====================================================================================================================
#define X_MAX_FILES 64
struct XCount {                      // kept records, their CIGAR ops, their own sequence blocks, the read groups they start
    uint32_t rec, ops, blk, grp;
    uint32_t of(DsCount c) const { return c == DS_RECS ? rec : c == DS_OPS ? ops : blk; }
};
struct XPlan {                       // per (source, destination): where the pieces of each file go
    uint32_t n_files;
    uint32_t mark_aln[X_MAX_FILES + 1];                                   // first local record of file f
    XCount dst[X_MAX_FILES];                                              // position in the destination's dataset
};

__global__ void k_x_touch(const uint32_t* __restrict__ contig, const uint32_t* __restrict__ read_id, uint64_t n, const uint32_t* __restrict__ owner,
                          uint32_t n_total, uint32_t* __restrict__ touch) {
    for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) {
        const uint32_t c = contig[i];
        const uint32_t o = (c == PP_CONTIG_UNKNOWN || c >= n_total) ? 0u : owner[c];      // unknown RNAMEs stay with shard 0 (shard.cpp)
        atomicOr(&touch[read_id[i]], 1u << o);
    }
}

// kept record -> (1, its ops, its own sequence blocks, 1 if it starts a group); element n is the scans' total slot.  `read0` is always 0
// (read ids are local to the source): ptxas gives the kernel two more registers without the subtraction.
__global__ void k_x_flags(const uint32_t* __restrict__ read_id, const uint16_t* __restrict__ n_cigar, const uint16_t* __restrict__ seq_len,
                          const uint8_t* __restrict__ flags, uint64_t n, uint32_t read0, const uint32_t* __restrict__ touch, uint32_t dest,
                          uint32_t* __restrict__ f_rec, uint32_t* __restrict__ f_ops, uint32_t* __restrict__ f_blk, uint32_t* __restrict__ f_grp) {
    for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i <= n; i += (uint64_t)gridDim.x * blockDim.x) {
        uint32_t r = 0, o = 0, b = 0, g = 0;
        if (i < n && ((touch[read_id[i] - read0] >> dest) & 1u)) {
            r = 1; o = n_cigar[i];
            if (!(flags[i] & (PP_FLAG_SEQSTAR | PP_FLAG_NOSEQ))) b = ((uint32_t)seq_len[i] + PP_SEQ_BLOCK - 1) / PP_SEQ_BLOCK;
            g = (i == 0 || read_id[i] != read_id[i - 1]) ? 1u : 0u;
        }
        f_rec[i] = r; f_ops[i] = o; f_blk[i] = b; f_grp[i] = g;
    }
}

__global__ void k_x_marks(const uint32_t* __restrict__ s_rec, const uint32_t* __restrict__ s_ops, const uint32_t* __restrict__ s_blk,
                          const uint32_t* __restrict__ s_grp, XPlan plan, XCount* __restrict__ out) {
    const uint32_t f = threadIdx.x;
    if (f <= plan.n_files) {
        const uint32_t i = plan.mark_aln[f];
        out[f] = XCount{s_rec[i], s_ops[i], s_blk[i], s_grp[i]};
    }
}

// records that own their sequence: where its first block goes (indexed by the OLD block offset, local to this source)
__global__ void k_x_blockmap(DsArrays a, uint64_t n, const uint32_t* __restrict__ s_rec, const uint32_t* __restrict__ s_blk, uint32_t* __restrict__ blockmap) {
    for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) {
        if (s_rec[i + 1] == s_rec[i]) continue;                                        // not kept
        if (a.flags[i] & (PP_FLAG_SEQSTAR | PP_FLAG_NOSEQ)) continue;
        blockmap[a.seq_off[i]] = s_blk[i];
    }
}

__global__ void k_x_pack(DsArrays a, DsArrays st, uint64_t n, XPlan plan, const uint32_t* __restrict__ s_rec, const uint32_t* __restrict__ s_ops,
                         const uint32_t* __restrict__ s_blk, const uint32_t* __restrict__ s_grp, const uint32_t* __restrict__ blockmap,
                         const XCount* __restrict__ marks /* scans at the file starts */) {
    for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) {
        const uint32_t j = s_rec[i];
        if (s_rec[i + 1] == j) continue;                                               // not kept
        uint32_t f = 0;
        while (f + 1 < plan.n_files && i >= plan.mark_aln[f + 1]) ++f;
        const uint32_t m_ops = marks[f].ops, m_blk = marks[f].blk, m_grp = marks[f].grp;
        const uint8_t fl = a.flags[i];
        const bool starts = (i == 0 || a.read_id[i] != a.read_id[i - 1]);
        st.contig[j] = a.contig[i]; st.ref_start[j] = a.ref_start[i]; st.nm[j] = a.nm[i];
        st.seq_len[j] = a.seq_len[i]; st.n_cigar[j] = a.n_cigar[i]; st.flags[j] = fl;
        st.read_id[j] = plan.dst[f].grp + (s_grp[i] + (starts ? 1u : 0u) - 1u - m_grp);
        st.cigar_off[j] = plan.dst[f].ops + (s_ops[i] - m_ops);
        uint32_t so = 0;
        if (!(fl & PP_FLAG_NOSEQ)) so = plan.dst[f].blk + (blockmap[a.seq_off[i]] - m_blk);
        st.seq_off[j] = so;
        const uint32_t nc = a.n_cigar[i], co = a.cigar_off[i];
        for (uint32_t t = 0; t < nc; ++t) st.cigar_ops[s_ops[i] + t] = a.cigar_ops[co + t];
    }
}

// the sequence blocks of kept owners, 16 bytes per thread
__global__ void k_x_pack_seq(DsArrays a, DsArrays st, uint64_t n, uint32_t blk_bytes, const uint32_t* __restrict__ s_rec, const uint32_t* __restrict__ s_blk) {
    const uint32_t per = blk_bytes / 16;
    for (uint64_t i = blockIdx.x * (uint64_t)(blockDim.x / 8) + threadIdx.x / 8; i < n; i += (uint64_t)gridDim.x * (blockDim.x / 8)) {
        if (s_rec[i + 1] == s_rec[i]) continue;
        const uint32_t nb = s_blk[i + 1] - s_blk[i];                                   // 0 for records without their own sequence
        if (!nb) continue;
        const uint4* src = reinterpret_cast<const uint4*>(a.seq_pool + (size_t)a.seq_off[i] * blk_bytes);
        uint4* dst = reinterpret_cast<uint4*>(st.seq_pool + (size_t)s_blk[i] * blk_bytes);
        for (uint32_t q = threadIdx.x & 7; q < nb * per; q += 8) dst[q] = src[q];
    }
}

struct TokState::XState {            // one context's tokenised ranges, moved out of the dataset buffers (same layout), as a source
    DevBuf b[DS_N];
    DevBuf stage[DS_N], touch, fl[4], sc[4], blockmap, marks, cubtmp;
    uint64_t n = 0, ops = 0, blk = 0, reads = 0;
    std::vector<TokState::Mark> mk;
    DevBuf d_owner;
    XCount* h_marks = nullptr;       // pinned
    void release() { for (auto& x : b) x.release(); for (auto& x : stage) x.release(); touch.release(); for (auto& x : fl) x.release();
                     for (auto& x : sc) x.release(); blockmap.release(); marks.release(); cubtmp.release(); d_owner.release();
                     if (h_marks) cudaFreeHost(h_marks); h_marks = nullptr; }
};
static void free_xstate(TokState* T) { if (T->xs) { T->xs->release(); delete T->xs; T->xs = nullptr; } }
namespace {
typedef TokState::XState XSource;

struct XSide {                       // one context of pp_tok_exchange_finish
    pp_ctx* ctx = nullptr;
    XSource* x = nullptr;
    std::vector<XCount> cnt;         // [destination * n_files + file]: what this source sends
    std::vector<XPlan> plan;         // [destination]
};

unsigned x_grid(const XSide& X) { return (unsigned)std::min<uint64_t>((X.x->n + 256) / 256 + 1, (uint64_t)X.ctx->sm_count * 32); }
}  // namespace

// The tokenised ranges of every context leave its dataset buffers (those receive the shard).  PP_TOK_HOST past the file limit.
static int x_take(std::vector<XSide>& S, pp_ctx* const* ctxs, int seq_bits, size_t* n_files, uint64_t* total_aln) {
    for (size_t g = 0; g < S.size(); ++g) {
        pp_ctx* ctx = ctxs[g];
        TokState* T = ctx->tok;
        if (!T || !T->active || T->marks.size() < 2 || T->seq_bits != seq_bits) return ctxs[0]->fail(PP_ERR_ARG, "pp_tok_exchange_finish: a context without tokenised ranges");
        if (g == 0) *n_files = T->marks.size() - 1;
        if (T->marks.size() - 1 != *n_files || *n_files > X_MAX_FILES) return PP_TOK_HOST;
        if (!T->xs) T->xs = new XSource();
        XSource& x = *T->xs;
        x.n = T->aln_base; x.ops = T->ops_base; x.blk = T->blk_base; x.reads = T->read_base; x.mk = T->marks;
        for (int k = 0; k < DS_N; ++k) std::swap(x.b[k], ctx->b[B_CONTIG + k]);
        *total_aln += x.n;
        XPlan P;
        memset(&P, 0, sizeof P);
        P.n_files = (uint32_t)*n_files;
        for (size_t f = 0; f <= *n_files; ++f) P.mark_aln[f] = (uint32_t)x.mk[f].aln;
        S[g].ctx = ctx; S[g].x = &x; S[g].plan.assign(S.size(), P);
    }
    return PP_OK;
}

// Source X's records bound for destination o: their flags (k_x_flags), the four exclusive scans over them, and the scans at the file
// starts (k_x_marks, into X's marks).  Both passes run it.
static int x_scan(XSide& X, int o) {
    pp_ctx* ctx = X.ctx;
    XSource& x = *X.x;
    cudaStream_t st = ctx->stream;
    const DsArrays A = ds_view(x.b);
    uint32_t* fl[4] = {x.fl[0].as<uint32_t>(), x.fl[1].as<uint32_t>(), x.fl[2].as<uint32_t>(), x.fl[3].as<uint32_t>()};
    uint32_t* sc[4] = {x.sc[0].as<uint32_t>(), x.sc[1].as<uint32_t>(), x.sc[2].as<uint32_t>(), x.sc[3].as<uint32_t>()};
    k_x_flags<<<x_grid(X), 256, 0, st>>>(A.read_id, A.n_cigar, A.seq_len, A.flags, x.n, 0u, x.touch.as<uint32_t>(), (uint32_t)o, fl[0], fl[1], fl[2], fl[3]);
    for (int k = 0; k < 4; ++k) {
        size_t tb = x.cubtmp.cap;
        CK(cub::DeviceScan::ExclusiveSum(x.cubtmp.p, tb, fl[k], sc[k], (int64_t)(x.n + 1), st));
    }
    k_x_marks<<<1, X_MAX_FILES + 1, 0, st>>>(sc[0], sc[1], sc[2], sc[3], X.plan[(size_t)o], x.marks.as<XCount>());
    return PP_OK;
}

// Pass one, on source X (context g): the destinations of every read group (k_x_touch), then what each destination gets out of each file.
static int x_count(XSide& X, int g, const uint32_t* owner, uint32_t n_total, size_t n_files) {
    pp_ctx* ctx = X.ctx;
    XSource& x = *X.x;
    cudaStream_t st = ctx->stream;
    const uint64_t n = x.n;
    const int n_ctx = (int)X.plan.size();
    CK(x.d_owner.ensure((size_t)n_total * 4 + 16));
    CK(cudaMemcpyAsync(x.d_owner.p, owner, (size_t)n_total * 4, cudaMemcpyHostToDevice, st));
    CK(x.touch.ensure((size_t)x.reads * 4 + 16));
    CK(cudaMemsetAsync(x.touch.p, 0, (size_t)x.reads * 4 + 16, st));
    for (int k = 0; k < 4; ++k) { CK(x.fl[k].ensure((n + 2) * 4)); CK(x.sc[k].ensure((n + 2) * 4)); }
    CK(x.marks.ensure((X_MAX_FILES + 1) * sizeof(XCount)));
    size_t tb = 0;
    CK(cub::DeviceScan::ExclusiveSum(nullptr, tb, (const uint32_t*)nullptr, (uint32_t*)nullptr, (int64_t)(n + 1), st));
    CK(x.cubtmp.ensure(tb + 256));
    const DsArrays A = ds_view(x.b);
    if (n) k_x_touch<<<x_grid(X), 256, 0, st>>>(A.contig, A.read_id, n, x.d_owner.as<uint32_t>(), n_total, x.touch.as<uint32_t>());
    X.cnt.assign((size_t)n_ctx * n_files, XCount{});
    for (int oo = 0; oo < n_ctx; ++oo) {
        const int o = (g + oo) % n_ctx;                                                // (the sources start on different destinations)
        const int rc = x_scan(X, o);
        if (rc != PP_OK) return rc;
        CK(cudaMemcpyAsync(x.h_marks, x.marks.p, (n_files + 1) * sizeof(XCount), cudaMemcpyDeviceToHost, st));
        CK(cudaStreamSynchronize(st));
        for (size_t f = 0; f < n_files; ++f) {
            const XCount &a = x.h_marks[f], &b = x.h_marks[f + 1];
            X.cnt[(size_t)o * n_files + f] = XCount{b.rec - a.rec, b.ops - a.ops, b.blk - a.blk, b.grp - a.grp};
        }
    }
    return PP_OK;
}

// On the host: at destination o, file by file, the pieces of the sources in order - global SAM order is (file, range, line), which is
// what the ordered depth needs.  Every destination's dataset buffers are sized for what it receives.  PP_TOK_HOST past the size limits.
static int x_plan(std::vector<XSide>& S, size_t n_files, int seq_bits) {
    for (size_t o = 0; o < S.size(); ++o) {
        uint64_t rec = 0, ops = 0, blk = 0, grp = 0;
        for (size_t f = 0; f < n_files; ++f)
            for (XSide& X : S) {
                X.plan[o].dst[f] = XCount{(uint32_t)rec, (uint32_t)ops, (uint32_t)blk, (uint32_t)grp};
                const XCount& c = X.cnt[o * n_files + f];
                rec += c.rec; ops += c.ops; blk += c.blk; grp += c.grp;
            }
        if (rec >= 0x7FFFFFFFull - 4096 || ops > 0xFFFFFFFFull || blk > 0xFFFFFFFFull || grp >= 0xFFFFFFFFull) return PP_TOK_HOST;
        pp_ctx* ctx = S[o].ctx;
        CK(cudaSetDevice(ctx->device));
        const uint64_t cnt[3] = {rec, ops, blk};
        for (int k = 0; k < DS_N; ++k) CK(ctx->b[B_CONTIG + k].ensure(ds_bytes(k, cnt, seq_bits) + 256));
        TokState* T = ctx->tok;
        T->aln_base = rec; T->ops_base = ops; T->blk_base = blk; T->read_base = grp;
    }
    return PP_OK;
}

// Pass two, on source X (context g): per destination the kept records compacted into the staging arrays with every offset renumbered
// for its place there (k_x_blockmap, k_x_pack, k_x_pack_seq), then each file's piece - one contiguous run of the staging arrays -
// copied into the destination's dataset.
static int x_send(XSide& X, int g, const std::vector<XSide>& S, size_t n_files, int seq_bits) {
    pp_ctx* ctx = X.ctx;
    XSource& x = *X.x;
    cudaStream_t st = ctx->stream;
    const uint64_t n = x.n;
    const uint64_t cnt[3] = {n, x.ops, x.blk};
    for (int k = 0; k < DS_N; ++k) CK(x.stage[k].ensure(ds_bytes(k, cnt, seq_bits) + 256));
    CK(x.blockmap.ensure((size_t)x.blk * 4 + 16));
    const DsArrays A = ds_view(x.b), Z = ds_view(x.stage);
    const uint32_t* sc[4] = {x.sc[0].as<uint32_t>(), x.sc[1].as<uint32_t>(), x.sc[2].as<uint32_t>(), x.sc[3].as<uint32_t>()};
    const int n_ctx = (int)S.size();
    for (int oo = 0; oo < n_ctx; ++oo) {
        const int o = (g + oo) % n_ctx;
        int rc = x_scan(X, o);
        if (rc != PP_OK) return rc;
        const XPlan& P = X.plan[(size_t)o];
        if (n) {
            k_x_blockmap<<<x_grid(X), 256, 0, st>>>(A, n, sc[0], sc[2], x.blockmap.as<uint32_t>());
            k_x_pack<<<x_grid(X), 256, 0, st>>>(A, Z, n, P, sc[0], sc[1], sc[2], sc[3], x.blockmap.as<uint32_t>(), x.marks.as<XCount>());
            k_x_pack_seq<<<(unsigned)std::min<uint64_t>((n + 31) / 32 + 1, (uint64_t)ctx->sm_count * 64), 256, 0, st>>>(A, Z, n, ds_block_bytes(seq_bits),
                                                                                                               sc[0], sc[2]);
        }
        CK(cudaMemcpyAsync(x.h_marks, x.marks.p, (n_files + 1) * sizeof(XCount), cudaMemcpyDeviceToHost, st));
        CK(cudaStreamSynchronize(st));
        pp_ctx* dctx = S[(size_t)o].ctx;
        for (size_t f = 0; f < n_files; ++f)
            for (int k = 0; k < DS_N; ++k) {
                const DsCount c = DS_ARRAYS[k].count;
                const size_t w = ds_width(k, seq_bits);
                const uint64_t from = x.h_marks[f].of(c), to = P.dst[f].of(c);
                rc = fx_copy(ctx, dctx, dctx->b[B_CONTIG + k].as<uint8_t>() + to * w, x.stage[k].as<uint8_t>() + from * w, (x.h_marks[f + 1].of(c) - from) * w);
                if (rc != PP_OK) return rc;
            }
        CK(cudaStreamSynchronize(st));                                                 // (the staging arrays are reused for the next destination)
    }
    return PP_OK;
}

static int x_exchange(pp_ctx* const* ctxs, int n_ctx, const uint32_t* owner, uint32_t n_total, const uint32_t* const* local_of,
                      const pp_contigs* shard_contigs, uint64_t* n_aln_total) {
    std::vector<XSide> S((size_t)n_ctx);
    const int seq_bits = ctxs[0]->tok ? ctxs[0]->tok->seq_bits : 4;
    size_t n_files = 0;
    uint64_t total_aln = 0;
    int rc = x_take(S, ctxs, seq_bits, &n_files, &total_aln);
    if (rc != PP_OK) return rc;
    for (XSide& X : S) {
        pp_ctx* ctx = X.ctx;
        CK(cudaSetDevice(ctx->device));
        if (!X.x->h_marks) CK(cudaHostAlloc((void**)&X.x->h_marks, (X_MAX_FILES + 1) * sizeof(XCount), cudaHostAllocDefault));
        enable_peers(ctx, ctxs, (size_t)n_ctx);
    }
    // every source works through its destinations on its own stream, driven by its own host thread
    if ((rc = fx_all(S, [&](XSide& X, int g) { return x_count(X, g, owner, n_total, n_files); })) != PP_OK) return rc;
    if ((rc = x_plan(S, n_files, seq_bits)) != PP_OK) return rc;
    if ((rc = fx_all(S, [&](XSide& X, int g) { return x_send(X, g, S, n_files, seq_bits); })) != PP_OK) return rc;
    if (n_aln_total) *n_aln_total = total_aln;
    // every GPU holds its groups in global SAM order: ghosts, the shard's contigs, binning
    for (int o = 0; o < n_ctx; ++o) {
        pp_ctx* ctx = ctxs[o];
        if (cudaSetDevice(ctx->device) != cudaSuccess) return PP_ERR_CUDA;
        rc = pp_tok_set_shard(ctx, local_of[o], n_total, &shard_contigs[o], o == 0);
        if (rc == PP_OK) rc = pp_tok_finish(ctx);
        if (rc != PP_OK) { if (ctx != ctxs[0]) ctxs[0]->err = ctx->err; return rc; }
    }
    return PP_OK;
}

extern "C" int pp_tok_exchange_finish(pp_ctx* const* ctxs, int n_ctx, const uint32_t* owner, uint32_t n_total, const uint32_t* const* local_of,
                                      const pp_contigs* shard_contigs, uint64_t* n_aln_total) {
    if (!ctxs || n_ctx < 1 || !owner || !local_of || !shard_contigs) return PP_ERR_ARG;
    if (n_ctx > 32) return PP_TOK_HOST;                                                // (one bit per destination in a group's mask: the host sharder takes over)
    const int rc = x_exchange(ctxs, n_ctx, owner, n_total, local_of, shard_contigs, n_aln_total);
    // (the buffers stay with the context: the range arrays that were swapped out are the spare capacity of the next call)
    if (rc != PP_OK)
        for (int g = 0; g < n_ctx; ++g)
            if (ctxs[g]->tok) ctxs[g]->tok->active = false;
    return rc;
}

// ---- the resident dataset, read back (tests compare it with the host packer's arrays)
extern "C" int pp_dataset_sizes(pp_ctx* ctx, pp_alignments* out) {
    if (!ctx || !out) return PP_ERR_ARG;
    if (!ctx->have_ds) return ctx->fail(PP_ERR_ARG, "pp_dataset_sizes: no resident dataset");
    memset(out, 0, sizeof *out);
    out->n_aln = ctx->n_aln; out->n_reads = ctx->n_reads; out->n_cigar_ops = ctx->n_ops; out->seq_pool_bytes = ctx->seq_bytes;
    out->seq_bits = ctx->seq_bits;
    return PP_OK;
}

extern "C" int pp_dataset_download(pp_ctx* ctx, const pp_alignments* into) {
    if (!ctx || !into) return PP_ERR_ARG;
    if (!ctx->have_ds) return ctx->fail(PP_ERR_ARG, "pp_dataset_download: no resident dataset");
    if (into->n_aln != ctx->n_aln || into->n_cigar_ops != ctx->n_ops || into->seq_pool_bytes != ctx->seq_bytes)
        return ctx->fail(PP_ERR_ARG, "pp_dataset_download: sizes differ from pp_dataset_sizes");
    CK(cudaSetDevice(ctx->device));
    cudaStream_t s = ctx->stream;
    const void* host[DS_N];
    ds_host(into, host);
    const uint64_t cnt[3] = {ctx->n_aln, ctx->n_ops, 0};
    for (int k = 0; k < DS_N; ++k) {
        const size_t bytes = k == DS_SEQPOOL ? (size_t)ctx->seq_bytes : ds_bytes(k, cnt, ctx->seq_bits);   // (an uploaded pool may end inside a block)
        if (host[k] && bytes) CK(cudaMemcpyAsync(const_cast<void*>(host[k]), ctx->b[B_CONTIG + k].p, bytes, cudaMemcpyDeviceToHost, s));
    }
    CK(cudaStreamSynchronize(s));
    return PP_OK;
}

// =====================================================================================================================
// `polypolish filter` on SAM text in HBM (SURVEY.md §8f-2): both files are streamed in, parsed (Alignment::new_quick,
// alignment.rs:102-128), their QNAMEs and RNAMEs interned in one device hash table (the reference's
// HashMap<String, Vec<Alignment>> keys, filter.rs:110-145), the filter proper runs on the arrays where they are
// (filter_kernels.cu), and the output SAM text (filter_sam, filter.rs:296-349: every line verbatim, "\tZP:Z:fail" appended to
// failing aligned records, '\n' line ends) is assembled on the device and streamed back into the output files.
// Anything unusual (a line the quick parse rejects, a file without alignments, a 64-bit hash collision between different
// strings, a size limit) answers PP_TOK_HOST and filter_pack.cpp does the job on the host, with the reference's messages.
// =====================================================================================================================
#include "filter_dev.h"

namespace {

struct FileDev {                       // one SAM file on the device
    const uint8_t* text;
    uint64_t n, n_lines;
    int unterminated;
    const unsigned long long* line_start;   // [n_lines + 1]
    tok::FLineRec* recs;                    // [n_lines]
    unsigned long long* s_al;               // [n_lines + 1] exclusive scan of "aligned"
    uint32_t *name_slot, *ref_slot;         // [n_lines] interned ids (aligned lines)
};

struct InternTable {
    unsigned long long* key;           // [cap] 0 = empty
    unsigned long long* rep;           // [cap] smallest (kind << 62 | file << 40 | line) that claimed the slot
    uint32_t mask;
};

struct FStatus {
    unsigned long long first_bad[2];   // per file: smallest line index the quick parse leaves to the host
    unsigned int collision;            // different strings with one 64-bit key, or a full table
    unsigned int pad;
};

__device__ __forceinline__ void fline_span(const FileDev& f, tok::Txt& x, uint64_t i, uint64_t& s, uint64_t& e) {
    s = f.line_start[i];
    if (i + 1 == f.n_lines && f.unterminated) { e = f.n; return; }
    e = f.line_start[i + 1] - 1;
    if (e > s && x.at(e - 1) == '\r') e--;
}

__global__ void __launch_bounds__(TK_LINE_THREADS) k_ftok_parse(FileDev f, int which, FStatus* st) {
    const uint64_t i = (uint64_t)blockIdx.x * TK_LINE_THREADS + threadIdx.x;
    if (i > f.n_lines) return;
    if (i == f.n_lines) { f.s_al[i] = 0; return; }
    tok::Txt x(f.text);
    uint64_t s, e;
    fline_span(f, x, i, s, e);
    tok::FLineRec r;
    const uint8_t kind = tok::parse_line_quick(x, s, e, r);
    r.kind = kind;
    f.recs[i] = r;
    f.s_al[i] = kind == tok::FK_ALIGNED ? 1 : 0;
    if (kind == tok::FK_HOST) atomicMin(&st->first_bad[which], (unsigned long long)i);
}

constexpr unsigned long long REF_DOMAIN = 0x9E3779B97F4A7C15ull;

// Claims the slot of `key` (insert-only linear probing: a key sits in the first slot of its probe sequence that was empty
// when it arrived, and slots never empty again, so every later arrival of the same key finds it).
__device__ __forceinline__ uint32_t intern(const InternTable& t, unsigned long long key, unsigned long long who, FStatus* st) {
    if (key == 0) key = 1;
    uint32_t sl = (uint32_t)(key ^ (key >> 32)) & t.mask;
    for (uint32_t probes = 0; probes <= t.mask; ++probes, sl = (sl + 1) & t.mask) {
        unsigned long long cur = t.key[sl];
        if (cur == 0) cur = atomicCAS(&t.key[sl], 0ull, key);
        if (cur == 0 || cur == key) {
            if (t.rep[sl] > who) atomicMin(&t.rep[sl], who);
            return sl;
        }
    }
    st->collision = 1;                 // table full
    return 0;
}

__global__ void __launch_bounds__(TK_LINE_THREADS) k_ftok_intern(FileDev f, int which, InternTable t, FStatus* st) {
    const uint64_t i = (uint64_t)blockIdx.x * TK_LINE_THREADS + threadIdx.x;
    if (i >= f.n_lines) return;
    const tok::FLineRec r = f.recs[i];
    if (r.kind != tok::FK_ALIGNED) return;
    const unsigned long long who = ((unsigned long long)which << 40) | i;
    f.name_slot[i] = intern(t, r.name_hash, who, st);
    f.ref_slot[i] = intern(t, r.ref_hash ^ REF_DOMAIN, (1ull << 62) | who, st);
}

// Every record confirms, byte by byte, that the string that owns its slot is its own string.
__global__ void __launch_bounds__(TK_LINE_THREADS) k_ftok_verify(FileDev f0, FileDev f1, int which, InternTable t, FStatus* st) {
    const FileDev& f = which ? f1 : f0;
    const uint64_t i = (uint64_t)blockIdx.x * TK_LINE_THREADS + threadIdx.x;
    if (i >= f.n_lines) return;
    const tok::FLineRec r = f.recs[i];
    if (r.kind != tok::FK_ALIGNED) return;
    const uint64_t s = f.line_start[i];
    tok::Txt x(f.text);
    for (int kind = 0; kind < 2; ++kind) {
        const unsigned long long rep = t.rep[kind ? f.ref_slot[i] : f.name_slot[i]];
        const int rk = (int)(rep >> 62), rf = (int)((rep >> 40) & 1);
        const uint64_t rl = rep & ((1ull << 40) - 1);
        bool same = rk == kind;
        if (same) {
            const FileDev& g = rf ? f1 : f0;
            const tok::FLineRec q = g.recs[rl];
            const uint64_t qs = g.line_start[rl];
            tok::Txt y(g.text);
            if (kind == 0) same = q.name_len == r.name_len && tok::same_bytes(x, s, y, qs, r.name_len);
            else same = q.ref_len == r.ref_len && tok::same_bytes(x, s + r.ref_rel, y, qs + q.ref_rel, r.ref_len);
        }
        if (!same) st->collision = 1;
    }
}

struct MateOut { uint32_t *name_id, *contig, *ref_start, *ref_end; uint8_t* flags; };

__global__ void __launch_bounds__(TK_LINE_THREADS) k_ftok_emit(FileDev f, MateOut m) {
    const uint64_t i = (uint64_t)blockIdx.x * TK_LINE_THREADS + threadIdx.x;
    if (i >= f.n_lines) return;
    const tok::FLineRec r = f.recs[i];
    if (r.kind != tok::FK_ALIGNED) return;
    const uint64_t a = f.s_al[i];
    m.name_id[a] = f.name_slot[i];
    m.contig[a] = f.ref_slot[i];
    m.ref_start[a] = r.ref_start;
    m.ref_end[a] = r.ref_end;
    m.flags[a] = r.rev;
}

// filter_sam (filter.rs:296-349): bytes of every output line.
__global__ void __launch_bounds__(TK_LINE_THREADS) k_ftok_outlen(FileDev f, const uint8_t* __restrict__ pass, unsigned long long* __restrict__ out_off) {
    const uint64_t i = (uint64_t)blockIdx.x * TK_LINE_THREADS + threadIdx.x;
    if (i > f.n_lines) return;
    if (i == f.n_lines) { out_off[i] = 0; return; }
    tok::Txt x(f.text);
    uint64_t s, e;
    fline_span(f, x, i, s, e);
    const bool fail = f.recs[i].kind == tok::FK_ALIGNED && !pass[f.s_al[i]];
    out_off[i] = (e - s) + 1 + (fail ? 10 : 0);
}

// One warp per line: the line's bytes, the tag for failing records, '\n'.
__global__ void __launch_bounds__(256) k_ftok_copy(FileDev f, const uint8_t* __restrict__ pass, const unsigned long long* __restrict__ out_off,
                                                   uint8_t* __restrict__ out) {
    const uint64_t i = ((uint64_t)blockIdx.x * 256 + threadIdx.x) >> 5;
    const uint32_t lane = threadIdx.x & 31;
    if (i >= f.n_lines) return;
    uint64_t s = f.line_start[i], e;
    if (i + 1 == f.n_lines && f.unterminated) e = f.n;
    else { e = f.line_start[i + 1] - 1; if (e > s && f.text[e - 1] == '\r') e--; }
    const bool fail = f.recs[i].kind == tok::FK_ALIGNED && !pass[f.s_al[i]];
    uint8_t* d = out + out_off[i];
    const uint64_t len = e - s;
    for (uint64_t k = lane; k < len; k += 32) d[k] = f.text[s + k];
    if (fail) { if (lane < 10) d[len + lane] = (uint8_t)"\tZP:Z:fail"[lane]; }
    if (lane == 0) d[len + (fail ? 10 : 0)] = '\n';
}

}  // namespace

// Streams n device bytes into fd (the mirror image of upload_file): each thread copies its slices into its pinned slots and
// from there into the file.  `map` is the file mapped MAP_SHARED (page faults of different threads proceed in parallel,
// whereas write()s to one file serialise on its inode lock: 3 GB/s on tmpfs whatever the thread count); when the mapping
// could not be made, pwrite() is used.  The bytes land at [base, base + n) of the file (`map` maps the whole file).
// PP_OK / PP_ERR_IO / PP_ERR_CUDA.
static int download_file(int device, TokState* T, const uint8_t* src, int fd, uint8_t* map, uint64_t n, int* cuda_err, uint64_t base = 0) {
    const int R = T->readers;
    const uint64_t n_slices = (n + TK_SLOT - 1) / TK_SLOT;
    std::atomic<int> err{0}, cerr{0};
    auto work = [&](int r) {
        if (cudaSetDevice(device) != cudaSuccess) { err = 2; return; }
        uint64_t k = 0, prev_o = 0, prev_len = 0;
        bool have_prev = false;
        auto flush_prev = [&](int slot) -> bool {
            cudaError_t e = cudaEventSynchronize(T->rev[r][slot]);
            if (e != cudaSuccess) { cerr = (int)e; err = 2; return false; }
            if (map) { memcpy(map + base + prev_o, T->pin[r][slot], (size_t)prev_len); return true; }
            uint64_t put = 0;
            while (put < prev_len) {
                const ssize_t g = pwrite(fd, T->pin[r][slot] + put, (size_t)(prev_len - put), (off_t)(base + prev_o + put));
                if (g <= 0) { err = 1; return false; }
                put += (uint64_t)g;
            }
            return true;
        };
        for (uint64_t sl = (uint64_t)r; sl < n_slices && !err; sl += (uint64_t)R, ++k) {
            const int slot = (int)(k & 1);
            const uint64_t o = sl * TK_SLOT, len = std::min<uint64_t>(TK_SLOT, n - o);
            cudaError_t e = cudaMemcpyAsync(T->pin[r][slot], src + o, (size_t)len, cudaMemcpyDeviceToHost, T->rstream[r]);
            if (e == cudaSuccess) e = cudaEventRecord(T->rev[r][slot], T->rstream[r]);
            if (e != cudaSuccess) { cerr = (int)e; err = 2; return; }
            if (have_prev && !flush_prev(slot ^ 1)) return;
            prev_o = o; prev_len = len; have_prev = true;
        }
        if (have_prev && !err) flush_prev((int)((k - 1) & 1));
    };
    std::vector<std::thread> th;
    for (int r = 1; r < R; ++r) th.emplace_back(work, r);
    work(0);
    for (auto& t : th) t.join();
    *cuda_err = cerr.load();
    return err == 1 ? PP_ERR_IO : err == 2 ? PP_ERR_CUDA : PP_OK;
}

// The same bytes to a descriptor that only takes sequential writes (pipe, FIFO, character device): one thread, two pinned slots,
// the copy of slice i+1 in flight while slice i is written.  PP_OK / PP_ERR_IO / PP_ERR_CUDA.
static int download_stream(int device, TokState* T, const uint8_t* src, int fd, uint64_t n, int* cuda_err) {
    if (cudaSetDevice(device) != cudaSuccess) return PP_ERR_CUDA;
    const uint64_t n_slices = (n + TK_SLOT - 1) / TK_SLOT;
    auto put_all = [&](const uint8_t* p, uint64_t len) {
        uint64_t put = 0;
        while (put < len) {
            const ssize_t g = write(fd, p + put, (size_t)(len - put));
            if (g < 0 && errno == EINTR) continue;
            if (g <= 0) return false;
            put += (uint64_t)g;
        }
        return true;
    };
    uint64_t prev_len = 0;
    for (uint64_t sl = 0; sl <= n_slices; ++sl) {
        const int slot = (int)(sl & 1);
        if (sl < n_slices) {
            const uint64_t o = sl * TK_SLOT, len = std::min<uint64_t>(TK_SLOT, n - o);
            cudaError_t e = cudaMemcpyAsync(T->pin[0][slot], src + o, (size_t)len, cudaMemcpyDeviceToHost, T->rstream[0]);
            if (e == cudaSuccess) e = cudaEventRecord(T->rev[0][slot], T->rstream[0]);
            if (e != cudaSuccess) { *cuda_err = (int)e; return PP_ERR_CUDA; }
        }
        if (sl > 0) {
            const cudaError_t e = cudaEventSynchronize(T->rev[0][slot ^ 1]);
            if (e != cudaSuccess) { *cuda_err = (int)e; return PP_ERR_CUDA; }
            if (!put_all(T->pin[0][slot ^ 1], prev_len)) return PP_ERR_IO;
        }
        if (sl < n_slices) prev_len = std::min<uint64_t>(TK_SLOT, n - sl * TK_SLOT);
    }
    return PP_OK;
}

// Line index + quick parse of one file whose text is on the device.  Fills fd; PP_OK / PP_TOK_HOST / error.
static int ftok_lines(pp_ctx* ctx, TokState* T, int which, const uint8_t* text, uint64_t n, bool unterminated, DevBuf& lines, DevBuf& tmp, FStatus* d_st,
                      FileDev* fd, uint32_t* launches) {
    cudaStream_t s = ctx->stream;
    LineIndex li;
    const int rc = line_count(ctx, T, text, n, unterminated, &li);
    if (rc != PP_OK) return rc;
    const uint64_t n_lines = li.n_lines;
    if (n_lines == 0) return PP_TOK_HOST;
    TRY_ALLOC(lines.ensure((n_lines + 2) * 8));
    size_t off = 0;
    auto carve = [&](size_t bytes) { size_t o = off; off += (bytes + 255) & ~size_t(255); return o; };
    const size_t o_rec = carve(n_lines * sizeof(tok::FLineRec)), o_al = carve((n_lines + 1) * 8), o_ns = carve(n_lines * 4), o_rs = carve(n_lines * 4);
    TRY_ALLOC(tmp.ensure(off));
    uint8_t* b = tmp.as<uint8_t>();
    fd->text = text; fd->n = n; fd->n_lines = n_lines; fd->unterminated = unterminated ? 1 : 0;
    fd->line_start = lines.as<unsigned long long>();
    fd->recs = (tok::FLineRec*)(b + o_rec); fd->s_al = (unsigned long long*)(b + o_al);
    fd->name_slot = (uint32_t*)(b + o_ns); fd->ref_slot = (uint32_t*)(b + o_rs);
    line_starts(ctx, text, li, lines.as<unsigned long long>());
    k_ftok_parse<<<(unsigned)((n_lines + 1 + TK_LINE_THREADS - 1) / TK_LINE_THREADS), TK_LINE_THREADS, 0, s>>>(*fd, which, d_st);
    size_t cub_bytes = 0;
    CK(cub::DeviceScan::ExclusiveSum(nullptr, cub_bytes, fd->s_al, fd->s_al, (int64_t)(n_lines + 1)));
    CK(T->cub.ensure(cub_bytes + 256));
    {
        size_t tb = T->cub.cap;
        CK(cub::DeviceScan::ExclusiveSum(T->cub.p, tb, fd->s_al, fd->s_al, (int64_t)(n_lines + 1), s));
    }
    *launches += 7;
    return PP_OK;
}

struct TokFilterBufs {                 // device buffers of the filter text path, kept in the tokeniser state
    DevBuf lines[2], tmp[2], mate[2], table, out, status, passkeep;
    DevBuf fx_refs, fx_stage, fx_rx, fx_owner, fx_home;   // the filter over several contexts: see filter_exchange
};

static void free_filter_bufs(TokFilterBufs* b) {
    for (int k = 0; k < 2; ++k) { b->lines[k].release(); b->tmp[k].release(); b->mate[k].release(); }
    b->table.release(); b->out.release(); b->status.release(); b->passkeep.release();
    b->fx_refs.release(); b->fx_stage.release(); b->fx_rx.release(); b->fx_owner.release(); b->fx_home.release();
    delete b;
}

// The filter's verdict as the polish records' ZP flag (alignment.rs:72-74): alignment i of the file failed -> PP_FLAG_ZPFAIL.
__global__ void __launch_bounds__(256) k_apply_pass(uint8_t* __restrict__ flags, const uint8_t* __restrict__ pass, uint64_t n) {
    const uint64_t i = (uint64_t)blockIdx.x * 256 + threadIdx.x;
    if (i < n && !pass[i]) flags[i] |= PP_FLAG_ZPFAIL;
}

// =====================================================================================================================
// `polypolish filter` over several GPUs (pp_filter_files_device, n_ctx > 1).  GPU g reads byte range g of both files (cut between read
// groups, so `filter-polish` can hand the same ranges to the polish tokeniser), indexes, parses and interns its lines as above.
// A record's verdict (alignment_pass_qc, filter.rs:352-377) depends only on the set of alignments that share its read name, and
// the insert-size statistics are sums over names, so the work partitions by read name:
//   k_fx_refs / k_fx_ref_bytes  every GPU's distinct RNAME strings go to the host, which numbers them by string (exact, no hash
//                               trust) and sends back a local -> global table (k_fx_scatter)
//   k_fx_count                  per destination: records, distinct names, name bytes (destination = owner of the QNAME key)
//   k_fx_names / k_fx_recs      compact records and each distinct name once (key + bytes) into per-destination staging, already
//                               numbered for their place at the destination; peer copies move them
//   k_fx_intern / k_fx_verify   the owner interns the names it received and confirms byte by byte that one key is one string
//   k_fx_mates                  the owner's two Mate arrays; then filter_begin / filter_hist / filter_pass (filter_kernels.cu),
//                               with the pair counts and the radix-select histograms summed on the host between the kernels
//   k_fx_home                   the verdicts, copied back to the source GPU, land at (file, aligned index); each GPU then writes
//                               its piece of each output file at its offset (k_ftok_outlen / k_ftok_copy / download_file)
// =====================================================================================================================
namespace {

struct FxCount { unsigned long long names, bytes, recs[2]; };
struct FxPlan { unsigned long long stage_name, stage_byte, stage_rec[2], name_base, byte_base; };
struct FxName { unsigned long long key; uint32_t off, len; };             // a distinct QNAME: its key; its bytes at `off`
struct FxRec { uint32_t name, contig, start, end, src, flags; };          // flags: bit 0 reverse strand, bit 1 second file
struct FxRef { unsigned long long pos; uint32_t slot, len; };             // a distinct RNAME: file << 63 | text offset

__device__ __forceinline__ uint32_t fx_owner(unsigned long long key, uint32_t n) {
    key ^= key >> 31; key *= 0xBF58476D1CE4E5B9ull; key ^= key >> 29;
    return (uint32_t)((key >> 32) % n);
}

__device__ __forceinline__ unsigned long long fx_who(int which, uint64_t i) { return ((unsigned long long)which << 40) | i; }

__global__ void __launch_bounds__(TK_LINE_THREADS) k_fx_refs(FileDev f, int which, InternTable t, FxRef* out, unsigned long long* n_out, uint64_t cap) {
    const uint64_t i = (uint64_t)blockIdx.x * TK_LINE_THREADS + threadIdx.x;
    if (i >= f.n_lines) return;
    const tok::FLineRec r = f.recs[i];
    if (r.kind != tok::FK_ALIGNED) return;
    const uint32_t sl = f.ref_slot[i];
    if (t.rep[sl] != ((1ull << 62) | fx_who(which, i))) return;     // the first line of this RNAME
    const unsigned long long j = atomicAdd(n_out, 1ull);
    if (j < cap) out[j] = FxRef{((unsigned long long)which << 63) | (f.line_start[i] + r.ref_rel), sl, r.ref_len};
}

__global__ void __launch_bounds__(256) k_fx_ref_bytes(const FxRef* __restrict__ refs, uint64_t n, const unsigned long long* __restrict__ off,
                                                      const uint8_t* __restrict__ t0, const uint8_t* __restrict__ t1, uint8_t* __restrict__ out) {
    const uint64_t j = (uint64_t)blockIdx.x * 256 + threadIdx.x;
    if (j >= n) return;
    const FxRef r = refs[j];
    const uint8_t* t = (r.pos >> 63) ? t1 : t0;
    const uint64_t p = r.pos & ~(1ull << 63);
    for (uint32_t k = 0; k < r.len; ++k) out[off[j] + k] = t[p + k];
}

__global__ void __launch_bounds__(256) k_fx_scatter(const uint2* __restrict__ pairs, uint64_t n, uint32_t* __restrict__ slot_val) {
    const uint64_t j = (uint64_t)blockIdx.x * 256 + threadIdx.x;
    if (j < n) slot_val[pairs[j].x] = pairs[j].y;
}

__global__ void __launch_bounds__(TK_LINE_THREADS) k_fx_count(FileDev f, int which, InternTable t, uint32_t n_dst, FxCount* cnt) {
    const uint64_t i = (uint64_t)blockIdx.x * TK_LINE_THREADS + threadIdx.x;
    if (i >= f.n_lines) return;
    const tok::FLineRec r = f.recs[i];
    if (r.kind != tok::FK_ALIGNED) return;
    const uint32_t d = fx_owner(r.name_hash, n_dst);
    atomicAdd(&cnt[d].recs[which], 1ull);
    if (t.rep[f.name_slot[i]] == fx_who(which, i)) { atomicAdd(&cnt[d].names, 1ull); atomicAdd(&cnt[d].bytes, (unsigned long long)r.name_len); }
}

// Each distinct name once per source GPU: key and bytes to its owner's staging; slot_val[name slot] = its index at the owner.
__global__ void __launch_bounds__(TK_LINE_THREADS) k_fx_names(FileDev f, int which, InternTable t, uint32_t n_dst, const FxPlan* __restrict__ plan,
                                                              FxCount* at, FxName* __restrict__ names, uint8_t* __restrict__ bytes,
                                                              uint32_t* __restrict__ slot_val) {
    const uint64_t i = (uint64_t)blockIdx.x * TK_LINE_THREADS + threadIdx.x;
    if (i >= f.n_lines) return;
    const tok::FLineRec r = f.recs[i];
    if (r.kind != tok::FK_ALIGNED || t.rep[f.name_slot[i]] != fx_who(which, i)) return;
    const uint32_t d = fx_owner(r.name_hash, n_dst);
    const FxPlan p = plan[d];
    const unsigned long long j = atomicAdd(&at[d].names, 1ull), b = atomicAdd(&at[d].bytes, (unsigned long long)r.name_len);
    names[p.stage_name + j] = FxName{r.name_hash, (uint32_t)(p.byte_base + b), r.name_len};
    const uint64_t s = f.line_start[i];
    for (uint32_t k = 0; k < r.name_len; ++k) bytes[p.stage_byte + b + k] = f.text[s + k];
    slot_val[f.name_slot[i]] = (uint32_t)(p.name_base + j);
}

__global__ void __launch_bounds__(TK_LINE_THREADS) k_fx_recs(FileDev f, int which, uint32_t n_dst, const FxPlan* __restrict__ plan, FxCount* at,
                                                             const uint32_t* __restrict__ slot_val, FxRec* __restrict__ recs) {
    const uint64_t i = (uint64_t)blockIdx.x * TK_LINE_THREADS + threadIdx.x;
    if (i >= f.n_lines) return;
    const tok::FLineRec r = f.recs[i];
    if (r.kind != tok::FK_ALIGNED) return;
    const uint32_t d = fx_owner(r.name_hash, n_dst);
    const unsigned long long j = atomicAdd(&at[d].recs[which], 1ull);
    recs[plan[d].stage_rec[which] + j] = FxRec{slot_val[f.name_slot[i]], slot_val[f.ref_slot[i]], r.ref_start, r.ref_end, (uint32_t)f.s_al[i],
                                               (uint32_t)r.rev | ((uint32_t)which << 1)};
}

__global__ void __launch_bounds__(256) k_fx_intern(const FxName* __restrict__ names, uint64_t n, InternTable t, uint32_t* __restrict__ id, FStatus* st) {
    const uint64_t e = (uint64_t)blockIdx.x * 256 + threadIdx.x;
    if (e < n) id[e] = intern(t, names[e].key, e, st);
}

// Every received name confirms, byte by byte, that the name that owns its slot is the same string.
__global__ void __launch_bounds__(256) k_fx_verify(const FxName* __restrict__ names, uint64_t n, const uint8_t* __restrict__ bytes, InternTable t,
                                                   const uint32_t* __restrict__ id, FStatus* st) {
    const uint64_t e = (uint64_t)blockIdx.x * 256 + threadIdx.x;
    if (e >= n) return;
    const FxName a = names[e], b = names[t.rep[id[e]]];
    bool same = a.len == b.len;
    for (uint32_t k = 0; same && k < a.len; ++k) same = bytes[a.off + k] == bytes[b.off + k];
    if (!same) st->collision = 1;
}

__global__ void __launch_bounds__(256) k_fx_mates(const FxRec* __restrict__ recs, uint64_t n, const uint32_t* __restrict__ id, MateOut m) {
    const uint64_t j = (uint64_t)blockIdx.x * 256 + threadIdx.x;
    if (j >= n) return;
    const FxRec r = recs[j];
    m.name_id[j] = id[r.name];
    m.contig[j] = r.contig;
    m.ref_start[j] = r.start;
    m.ref_end[j] = r.end;
    m.flags[j] = (uint8_t)(r.flags & 1);
}

// The owners' verdicts, back in the staging order of this GPU, go to (file, aligned index).
__global__ void __launch_bounds__(256) k_fx_home(const FxRec* __restrict__ recs, uint64_t n, const uint8_t* __restrict__ ret, uint8_t* __restrict__ pass0,
                                                 uint8_t* __restrict__ pass1) {
    const uint64_t j = (uint64_t)blockIdx.x * 256 + threadIdx.x;
    if (j >= n) return;
    const FxRec r = recs[j];
    ((r.flags & 2) ? pass1 : pass0)[r.src] = ret[j];
}

unsigned fx_blocks(uint64_t n, unsigned per) { return (unsigned)((n + per - 1) / per); }

// One context of pp_filter_files_device: its text (the whole files, or one byte range of each) and, over several contexts, the
// records and names it sends as a source and the names it owns as an owner.
struct FilterSide {
    pp_ctx* ctx = nullptr;
    TokState* T = nullptr;
    TokFilterBufs* B = nullptr;
    FStatus* d_st = nullptr;
    FileDev fd[2];
    uint64_t n_al[2] = {0, 0};
    InternTable tb{};
    uint32_t* slot_val = nullptr;          // [table slots] after interning: global contig id (RNAME slots), index at the owner (QNAME slots)
    // as a source
    std::vector<FxRef> refs;
    std::vector<uint64_t> ref_off;
    std::vector<uint8_t> ref_bytes;
    std::vector<uint2> ref_global;
    std::vector<FxCount> cnt;              // [destination]
    std::vector<FxPlan> plan;              // [destination]
    uint64_t st_names = 0, st_bytes = 0, st_recs[2] = {0, 0};
    FxCount* d_at = nullptr;
    FxPlan* d_plan = nullptr;
    FxName* s_names = nullptr;
    uint8_t* s_bytes = nullptr;
    FxRec* s_recs = nullptr;
    uint8_t* ret = nullptr;                // [st_recs[0] + st_recs[1]] the owners' verdicts, staging order
    uint8_t* pass[2] = {nullptr, nullptr}; // [n_al[k]] verdicts by aligned index
    // as an owner
    uint64_t rx_names = 0, rx_bytes = 0, rx_recs[2] = {0, 0};
    FxName* r_names = nullptr;
    uint8_t* r_bytes = nullptr;
    FxRec* r_recs[2] = {nullptr, nullptr};
    FilterDev f{};
    unsigned long long pairs[4] = {0, 0, 0, 0}, np[2] = {0, 0};
    uint32_t hist[512];
    uint64_t out_n = 0;
    uint32_t launches = 0;
    float h2d_ms = 0;
    pp_tok_stats tst[2];
};

}  // namespace

// Text in, on one context: both texts into HBM, the second streaming in while the first is indexed and parsed (ftok_lines; an empty
// range is skipped), and the aligned counts.  With `cuts` the context reads bytes [cuts[f][g], cuts[f][g + 1]) of file f, else the
// whole files.  PP_OK, PP_TOK_HOST (a line the quick parse leaves to the host, a size limit) or an error.
static int fx_text_in(FilterSide& X, int g, const char* const ins[2], const uint64_t* const cuts[2]) {
    pp_ctx* ctx = X.ctx;
    TokState* T = X.T;
    TokFilterBufs& B = *X.B;
    cudaStream_t s = ctx->stream;
    CK(B.status.ensure(sizeof(FStatus)));
    X.d_st = B.status.as<FStatus>();
    FStatus h_st;
    h_st.first_bad[0] = h_st.first_bad[1] = ~0ull; h_st.collision = 0; h_st.pad = 0;
    CK(cudaMemcpyAsync(X.d_st, &h_st, sizeof h_st, cudaMemcpyHostToDevice, s));
    CK(cudaStreamSynchronize(s));
    if (cuts) {
        T->range_off = {cuts[0][g], cuts[1][g]};
        T->range_len = {cuts[0][g + 1] - cuts[0][g], cuts[1][g + 1] - cuts[1][g]};
    }
    for (int k = 0; k < 2; ++k) {
        int r = prefetch_wait(ctx, T, ins[k], false, cuts ? k : -1);
        if (r != PP_OK) return r;
        const uint64_t nb = T->pf.n;
        const uint8_t* text = T->text[T->pf.buf].as<uint8_t>();
        const bool unterminated = nb > 0 && T->pf.last != '\n';
        X.h2d_ms += T->pf.ms;
        if (k == 0 && (r = prefetch_start(ctx, T, ins[1], false, cuts ? 1 : -1)) != PP_OK) return r;
        FileDev& fd = X.fd[k];
        memset(&fd, 0, sizeof fd);
        fd.text = text;
        if (nb) r = ftok_lines(ctx, T, k, text, nb, unterminated, B.lines[k], B.tmp[k], X.d_st, &fd, &X.launches);
        if (r != PP_OK) {
            if (T->pf.active) { if (T->pf.th.joinable()) T->pf.th.join(); T->pf.active = false; }
            return r;
        }
    }
    for (int k = 0; k < 2; ++k)
        if (X.fd[k].n_lines) CK(cudaMemcpyAsync(T->h_tot + k, X.fd[k].s_al + X.fd[k].n_lines, 8, cudaMemcpyDeviceToHost, s));
    CK(cudaMemcpyAsync(&h_st, X.d_st, sizeof h_st, cudaMemcpyDeviceToHost, s));
    CK(cudaStreamSynchronize(s));
    CK(cudaGetLastError());
    for (int k = 0; k < 2; ++k) X.n_al[k] = X.fd[k].n_lines ? T->h_tot[k] : 0;
    if (h_st.first_bad[0] != ~0ull || h_st.first_bad[1] != ~0ull) return PP_TOK_HOST;
    if (X.n_al[0] >= 0x7FFFFFFFull || X.n_al[1] >= 0x7FFFFFFFull) return PP_TOK_HOST;
    return PP_OK;
}

// Local interning, on one context: every QNAME and RNAME of its text gets a slot of one table (k_ftok_intern), and every record
// confirms its slot's string byte by byte (k_ftok_verify, which flags a collision for the caller's next status read).
static int fx_intern(FilterSide& X) {
    pp_ctx* ctx = X.ctx;
    cudaStream_t s = ctx->stream;
    uint64_t cap = 1024;
    while (cap < 3 * (X.n_al[0] + X.n_al[1]) + 1024) cap <<= 1;
    if (cap > (1ull << 31)) return PP_TOK_HOST;
    TRY_ALLOC(X.B->table.ensure(cap * 16));
    X.tb.key = X.B->table.as<unsigned long long>(); X.tb.rep = X.tb.key + cap; X.tb.mask = (uint32_t)(cap - 1);
    CK(cudaMemsetAsync(X.tb.key, 0, cap * 8, s));
    CK(cudaMemsetAsync(X.tb.rep, 0xFF, cap * 8, s));
    for (int k = 0; k < 2; ++k)
        if (X.fd[k].n_lines) k_ftok_intern<<<fx_blocks(X.fd[k].n_lines, TK_LINE_THREADS), TK_LINE_THREADS, 0, s>>>(X.fd[k], k, X.tb, X.d_st);
    for (int k = 0; k < 2; ++k)
        if (X.fd[k].n_lines) k_ftok_verify<<<fx_blocks(X.fd[k].n_lines, TK_LINE_THREADS), TK_LINE_THREADS, 0, s>>>(X.fd[0], X.fd[1], k, X.tb, X.d_st);
    X.launches += 4;
    return PP_OK;
}

// The filter on one context: its mate arrays written straight from its lines (k_ftok_emit), then the whole filter on the device
// (pp_filter_core: the thresholds are picked there, no host round trips).  With `fuse` the verdicts move out of the context's
// scratch buffer, which the polish tokeniser uses next.
template <class Lap>
static int filter_one(FilterSide& X, const pp_filter_params* prm_in, pp_filter_result* res, bool fuse, Lap&& lap) {
    pp_ctx* ctx = X.ctx;
    TokFilterBufs& B = *X.B;
    cudaStream_t s = ctx->stream;
    int rc = fx_intern(X);
    if (rc != PP_OK) return rc;
    Mate mates[2];
    for (int k = 0; k < 2; ++k) {
        const size_t na = (size_t)X.n_al[k];
        TRY_ALLOC(B.mate[k].ensure(na * 17 + 5 * 256));
        uint8_t* mb = B.mate[k].as<uint8_t>();
        auto up = [](size_t v) { return (v + 255) & ~size_t(255); };
        MateOut mo;
        mo.name_id = (uint32_t*)mb; mo.contig = (uint32_t*)(mb + up(na * 4)); mo.ref_start = (uint32_t*)(mb + 2 * up(na * 4));
        mo.ref_end = (uint32_t*)(mb + 3 * up(na * 4)); mo.flags = mb + 4 * up(na * 4);
        k_ftok_emit<<<fx_blocks(X.fd[k].n_lines, TK_LINE_THREADS), TK_LINE_THREADS, 0, s>>>(X.fd[k], mo);
        mates[k].name_id = mo.name_id; mates[k].contig = mo.contig; mates[k].ref_start = mo.ref_start; mates[k].ref_end = mo.ref_end;
        mates[k].flags = mo.flags; mates[k].cnt = nullptr; mates[k].head = nullptr; mates[k].next = nullptr; mates[k].pass = nullptr;
        mates[k].n = (uint32_t)na;
    }
    X.launches += 2;
    FStatus h_st;
    CK(cudaMemcpyAsync(&h_st, X.d_st, sizeof h_st, cudaMemcpyDeviceToHost, s));
    CK(cudaStreamSynchronize(s));
    CK(cudaGetLastError());
    if (h_st.collision) return PP_TOK_HOST;
    lap(1);

    pp_filter_params prm = *prm_in;
    prm.n_names = X.tb.mask + 1ull;
    res->pass1 = nullptr; res->pass2 = nullptr;
    const uint8_t* d_pass[2] = {nullptr, nullptr};
    uint64_t np[2] = {0, 0};
    CK(cudaEventRecord(ctx->ev[0], s));
    rc = pp_filter_core(ctx, mates, &prm, res, d_pass, np);
    if (rc != PP_OK) return rc;
    X.launches += res->timing.launches;
    for (int k = 0; k < 2; ++k) { X.np[k] = np[k]; X.pass[k] = (uint8_t*)d_pass[k]; }
    if (fuse) {
        CK(B.passkeep.ensure(X.n_al[0] + X.n_al[1] + 64));
        uint8_t* keep = B.passkeep.as<uint8_t>();
        CK(cudaMemcpyAsync(keep, d_pass[0], X.n_al[0], cudaMemcpyDeviceToDevice, s));
        CK(cudaMemcpyAsync(keep + X.n_al[0], d_pass[1], X.n_al[1], cudaMemcpyDeviceToDevice, s));
        CK(cudaStreamSynchronize(s));
        X.pass[0] = keep; X.pass[1] = keep + X.n_al[0];
    }
    return PP_OK;
}

// The filter over several contexts (see the comment above the k_fx_ kernels): the records meet on the context that owns their read
// name, and the pair counts and the radix select's histograms are summed on the host.  The verdicts end up in every source's pass[k].
template <class Lap>
static int filter_exchange(std::vector<FilterSide>& S, const pp_filter_params* prm, pp_filter_result* res, Lap&& lap) {
    const uint32_t n = (uint32_t)S.size();
    // ---- every context: local interning, then its distinct RNAMEs with their bytes
    int rc = fx_all(S, [&](FilterSide& X, int) -> int {
        pp_ctx* ctx = X.ctx;
        TokState* T = X.T;
        TokFilterBufs& B = *X.B;
        cudaStream_t s = ctx->stream;
        int r = fx_intern(X);
        if (r != PP_OK) return r;
        X.slot_val = (uint32_t*)X.tb.key;                                   // (the keys are done with once the slots are verified)
        uint64_t rcap = std::max<uint64_t>(1024, B.fx_refs.cap / 2 / sizeof(FxRef));
        for (;;) {
            TRY_ALLOC(B.fx_refs.ensure(2 * rcap * sizeof(FxRef) + 64));
            FxRef* d_refs = B.fx_refs.as<FxRef>();
            unsigned long long* d_n = (unsigned long long*)(d_refs + 2 * rcap - 1);
            CK(cudaMemsetAsync(d_n, 0, 8, s));
            for (int k = 0; k < 2; ++k)
                if (X.fd[k].n_lines) k_fx_refs<<<fx_blocks(X.fd[k].n_lines, TK_LINE_THREADS), TK_LINE_THREADS, 0, s>>>(X.fd[k], k, X.tb, d_refs, d_n, rcap);
            FStatus h_st;
            CK(cudaMemcpyAsync(T->h_tot, d_n, 8, cudaMemcpyDeviceToHost, s));
            CK(cudaMemcpyAsync(&h_st, X.d_st, sizeof h_st, cudaMemcpyDeviceToHost, s));
            CK(cudaStreamSynchronize(s));
            CK(cudaGetLastError());
            if (h_st.collision) return PP_TOK_HOST;
            const uint64_t nr = T->h_tot[0];
            if (nr > rcap) { rcap = nr; continue; }
            X.refs.resize(nr);
            X.ref_off.assign(nr + 1, 0);
            if (nr) CK(cudaMemcpyAsync(X.refs.data(), d_refs, nr * sizeof(FxRef), cudaMemcpyDeviceToHost, s));
            CK(cudaStreamSynchronize(s));
            for (uint64_t j = 0; j < nr; ++j) X.ref_off[j + 1] = X.ref_off[j] + X.refs[j].len;
            X.ref_bytes.resize(X.ref_off[nr] + 1);
            if (nr) {
                unsigned long long* d_off = (unsigned long long*)(d_refs + nr);       // (second half of the buffer)
                uint8_t* d_bytes;
                TRY_ALLOC(B.fx_stage.ensure(X.ref_off[nr] + 64));
                d_bytes = B.fx_stage.as<uint8_t>();
                CK(cudaMemcpyAsync(d_off, X.ref_off.data(), nr * 8, cudaMemcpyHostToDevice, s));
                k_fx_ref_bytes<<<fx_blocks(nr, 256), 256, 0, s>>>(d_refs, nr, d_off, X.fd[0].text, X.fd[1].text, d_bytes);
                CK(cudaMemcpyAsync(X.ref_bytes.data(), d_bytes, X.ref_off[nr], cudaMemcpyDeviceToHost, s));
                CK(cudaStreamSynchronize(s));
                CK(cudaGetLastError());
            }
            break;
        }
        X.launches += 2;
        return PP_OK;
    });
    if (rc != PP_OK) return rc;
    lap(0);

    // ---- global RNAME ids: numbered by string, in the order the GPUs list them
    {
        std::unordered_map<std::string, uint32_t> global;
        for (FilterSide& X : S) {
            X.ref_global.resize(X.refs.size());
            for (size_t j = 0; j < X.refs.size(); ++j) {
                const std::string name((const char*)X.ref_bytes.data() + X.ref_off[j], X.refs[j].len);
                X.ref_global[j] = make_uint2(X.refs[j].slot, global.emplace(name, (uint32_t)global.size()).first->second);
            }
        }
    }
    // ---- count what goes where
    rc = fx_all(S, [&](FilterSide& X, int) -> int {
        pp_ctx* ctx = X.ctx;
        cudaStream_t s = ctx->stream;
        TokFilterBufs& B = *X.B;
        const uint64_t nr = X.ref_global.size();
        TRY_ALLOC(B.fx_stage.ensure(nr * sizeof(uint2) + 2 * n * (sizeof(FxCount) + sizeof(FxPlan)) + 256));
        uint2* d_pairs = B.fx_stage.as<uint2>();
        if (nr) {
            CK(cudaMemcpyAsync(d_pairs, X.ref_global.data(), nr * sizeof(uint2), cudaMemcpyHostToDevice, s));
            k_fx_scatter<<<fx_blocks(nr, 256), 256, 0, s>>>(d_pairs, nr, X.slot_val);
        }
        FxCount* d_cnt = (FxCount*)(B.fx_stage.as<uint8_t>() + ((nr * sizeof(uint2) + 255) & ~size_t(255)));
        CK(cudaMemsetAsync(d_cnt, 0, n * sizeof(FxCount), s));
        for (int k = 0; k < 2; ++k)
            if (X.fd[k].n_lines) k_fx_count<<<fx_blocks(X.fd[k].n_lines, TK_LINE_THREADS), TK_LINE_THREADS, 0, s>>>(X.fd[k], k, X.tb, n, d_cnt);
        X.cnt.resize(n);
        CK(cudaMemcpyAsync(X.cnt.data(), d_cnt, n * sizeof(FxCount), cudaMemcpyDeviceToHost, s));
        CK(cudaStreamSynchronize(s));
        CK(cudaGetLastError());
        X.launches += 3;
        return PP_OK;
    });
    if (rc != PP_OK) return rc;
    // where every piece goes: at destination d, the pieces of the sources in order; at source g, the destinations in order (file by file)
    for (uint32_t d = 0; d < n; ++d) {
        uint64_t at_names = 0, at_bytes = 0, at_recs[2] = {0, 0};
        for (uint32_t g = 0; g < n; ++g) {
            const FxCount& c = S[g].cnt[d];
            at_names += c.names; at_bytes += c.bytes; at_recs[0] += c.recs[0]; at_recs[1] += c.recs[1];
        }
        if (at_names >= 0x7FFFFFFFull || at_bytes >= 0xFFFFFFFFull) return PP_TOK_HOST;
        S[d].rx_names = at_names; S[d].rx_bytes = at_bytes; S[d].rx_recs[0] = at_recs[0]; S[d].rx_recs[1] = at_recs[1];
    }
    for (uint32_t g = 0; g < n; ++g) {
        FilterSide& X = S[g];
        X.plan.assign(n, FxPlan{});
        X.st_names = X.st_bytes = X.st_recs[0] = X.st_recs[1] = 0;
        for (uint32_t d = 0; d < n; ++d) {
            FxPlan& p = X.plan[d];
            p.stage_name = X.st_names; p.stage_byte = X.st_bytes;
            X.st_names += X.cnt[d].names; X.st_bytes += X.cnt[d].bytes;
            for (uint32_t h = 0; h < g; ++h) { p.name_base += S[h].cnt[d].names; p.byte_base += S[h].cnt[d].bytes; }
        }
        for (int k = 0; k < 2; ++k)
            for (uint32_t d = 0; d < n; ++d) { X.plan[d].stage_rec[k] = X.st_recs[0] + X.st_recs[1]; X.st_recs[k] += X.cnt[d].recs[k]; }
    }
    auto rec_base = [&](uint32_t g, uint32_t d, int k) { uint64_t b = 0; for (uint32_t h = 0; h < g; ++h) b += S[h].cnt[d].recs[k]; return b; };

    // ---- staging (source) and receive buffers (owner); then the pieces travel
    rc = fx_all(S, [&](FilterSide& X, int) -> int {
        pp_ctx* ctx = X.ctx;
        cudaStream_t s = ctx->stream;
        TokFilterBufs& B = *X.B;
        auto up = [](uint64_t v) { return (v + 255) & ~uint64_t(255); };
        const uint64_t st_recs = X.st_recs[0] + X.st_recs[1];
        const uint64_t o_plan = 0, o_at = up(n * sizeof(FxPlan)), o_names = o_at + up(n * sizeof(FxCount)), o_recs = o_names + up(X.st_names * sizeof(FxName)),
                       o_bytes = o_recs + up(st_recs * sizeof(FxRec));
        TRY_ALLOC(B.fx_stage.ensure(o_bytes + X.st_bytes + 64));
        uint8_t* b = B.fx_stage.as<uint8_t>();
        X.d_plan = (FxPlan*)(b + o_plan); X.d_at = (FxCount*)(b + o_at); X.s_names = (FxName*)(b + o_names); X.s_recs = (FxRec*)(b + o_recs);
        X.s_bytes = b + o_bytes;
        const uint64_t o_pass1 = up(X.n_al[0] + 1), o_ret = o_pass1 + up(X.n_al[1] + 1);
        TRY_ALLOC(B.fx_home.ensure(o_ret + st_recs + 64));
        X.pass[0] = B.fx_home.as<uint8_t>(); X.pass[1] = X.pass[0] + o_pass1; X.ret = X.pass[0] + o_ret;
        const uint64_t o_rb = up(X.rx_names * sizeof(FxName)), o_r0 = o_rb + up(X.rx_bytes + 1), o_r1 = o_r0 + up(X.rx_recs[0] * sizeof(FxRec));
        TRY_ALLOC(B.fx_rx.ensure(o_r1 + X.rx_recs[1] * sizeof(FxRec) + 64));
        uint8_t* r = B.fx_rx.as<uint8_t>();
        X.r_names = (FxName*)r; X.r_bytes = r + o_rb; X.r_recs[0] = (FxRec*)(r + o_r0); X.r_recs[1] = (FxRec*)(r + o_r1);
        CK(cudaMemcpyAsync(X.d_plan, X.plan.data(), n * sizeof(FxPlan), cudaMemcpyHostToDevice, s));
        CK(cudaMemsetAsync(X.d_at, 0, n * sizeof(FxCount), s));
        for (int k = 0; k < 2; ++k)
            if (X.fd[k].n_lines)
                k_fx_names<<<fx_blocks(X.fd[k].n_lines, TK_LINE_THREADS), TK_LINE_THREADS, 0, s>>>(X.fd[k], k, X.tb, n, X.d_plan, X.d_at, X.s_names,
                                                                                                  X.s_bytes, X.slot_val);
        for (int k = 0; k < 2; ++k)
            if (X.fd[k].n_lines)
                k_fx_recs<<<fx_blocks(X.fd[k].n_lines, TK_LINE_THREADS), TK_LINE_THREADS, 0, s>>>(X.fd[k], k, n, X.d_plan, X.d_at, X.slot_val, X.s_recs);
        CK(cudaStreamSynchronize(s));
        CK(cudaGetLastError());
        X.launches += 4;
        return PP_OK;
    });
    if (rc != PP_OK) return rc;
    rc = fx_all(S, [&](FilterSide& X, int g) -> int {
        for (uint32_t dd = 0; dd < n; ++dd) {
            const uint32_t d = ((uint32_t)g + dd) % n;                      // (the sources start on different destinations)
            FilterSide& D = S[d];
            const FxPlan& p = X.plan[d];
            const FxCount& c = X.cnt[d];
            int r = fx_copy(X.ctx, D.ctx, D.r_names + p.name_base, X.s_names + p.stage_name, c.names * sizeof(FxName));
            if (r == PP_OK) r = fx_copy(X.ctx, D.ctx, D.r_bytes + p.byte_base, X.s_bytes + p.stage_byte, c.bytes);
            for (int k = 0; k < 2 && r == PP_OK; ++k)
                r = fx_copy(X.ctx, D.ctx, D.r_recs[k] + rec_base((uint32_t)g, d, k), X.s_recs + p.stage_rec[k], c.recs[k] * sizeof(FxRec));
            if (r != PP_OK) return r;
        }
        pp_ctx* ctx = X.ctx;
        CK(cudaStreamSynchronize(ctx->stream));
        return PP_OK;
    });
    if (rc != PP_OK) return rc;
    lap(1);

    // ---- owners: intern and verify the names they received, their two Mate arrays, unique pairs
    rc = fx_all(S, [&](FilterSide& X, int) -> int {
        pp_ctx* ctx = X.ctx;
        cudaStream_t s = ctx->stream;
        TokFilterBufs& B = *X.B;
        uint64_t cap = 1024;
        while (cap < 2 * X.rx_names + 1024) cap <<= 1;
        if (cap > (1ull << 31)) return PP_TOK_HOST;
        auto up = [](uint64_t v) { return (v + 255) & ~uint64_t(255); };
        const uint64_t o_id = cap * 16, o_m = o_id + up(X.rx_names * 4 + 4);
        uint64_t o_mate[2][5], end = o_m;
        for (int k = 0; k < 2; ++k)
            for (int a = 0; a < 5; ++a) { o_mate[k][a] = end; end += up(X.rx_recs[k] * (a < 4 ? 4 : 1) + 4); }
        TRY_ALLOC(B.fx_owner.ensure(end + 64));
        uint8_t* b = B.fx_owner.as<uint8_t>();
        InternTable t;
        t.key = (unsigned long long*)b; t.rep = t.key + cap; t.mask = (uint32_t)(cap - 1);
        uint32_t* id = (uint32_t*)(b + o_id);
        CK(cudaMemsetAsync(t.key, 0, cap * 8, s));
        CK(cudaMemsetAsync(t.rep, 0xFF, cap * 8, s));
        if (X.rx_names) {
            k_fx_intern<<<fx_blocks(X.rx_names, 256), 256, 0, s>>>(X.r_names, X.rx_names, t, id, X.d_st);
            k_fx_verify<<<fx_blocks(X.rx_names, 256), 256, 0, s>>>(X.r_names, X.rx_names, X.r_bytes, t, id, X.d_st);
        }
        Mate mates[2];
        for (int k = 0; k < 2; ++k) {
            MateOut mo;
            mo.name_id = (uint32_t*)(b + o_mate[k][0]); mo.contig = (uint32_t*)(b + o_mate[k][1]); mo.ref_start = (uint32_t*)(b + o_mate[k][2]);
            mo.ref_end = (uint32_t*)(b + o_mate[k][3]); mo.flags = b + o_mate[k][4];
            if (X.rx_recs[k]) k_fx_mates<<<fx_blocks(X.rx_recs[k], 256), 256, 0, s>>>(X.r_recs[k], X.rx_recs[k], id, mo);
            mates[k].name_id = mo.name_id; mates[k].contig = mo.contig; mates[k].ref_start = mo.ref_start; mates[k].ref_end = mo.ref_end;
            mates[k].flags = mo.flags; mates[k].cnt = nullptr; mates[k].head = nullptr; mates[k].next = nullptr; mates[k].pass = nullptr;
            mates[k].n = (uint32_t)X.rx_recs[k];
        }
        X.launches += 4;
        CK(cudaEventRecord(ctx->ev[0], s));
        int r = filter_begin(ctx, mates, (uint32_t)cap, &X.f, &X.launches);
        if (r != PP_OK) return r;
        FStatus h_st;
        CK(cudaMemcpyAsync(X.pairs, X.f.pairs, 32, cudaMemcpyDeviceToHost, s));
        CK(cudaMemcpyAsync(&h_st, X.d_st, sizeof h_st, cudaMemcpyDeviceToHost, s));
        CK(cudaStreamSynchronize(s));
        CK(cudaGetLastError());
        return h_st.collision ? PP_TOK_HOST : PP_OK;
    });
    if (rc != PP_OK) return rc;

    // ---- orientation from the summed pair counts, thresholds by a radix select over all owners (filter.rs:148-186)
    unsigned long long pairs[4] = {0, 0, 0, 0};
    for (FilterSide& X : S) for (int i = 0; i < 4; ++i) pairs[i] += X.pairs[i];
    for (int i = 0; i < 4; ++i) res->pairs[i] = pairs[i];
    int chosen = 0;
    unsigned long long n_sizes = 0;
    rc = filter_orientation(S[0].ctx, prm, pairs, &chosen, &n_sizes);
    if (rc != PP_OK) return rc;
    res->orientation = chosen;
    bool in_range[2];
    unsigned long long rank[2];
    filter_ranks(prm, n_sizes, rank, in_range);
    uint32_t prefix[2] = {0, 0}, done_mask = 0;
    for (const int shift : FILTER_SHIFTS) {
        rc = fx_all(S, [&](FilterSide& X, int) { return filter_hist(X.ctx, X.f, (uint32_t)chosen, shift, done_mask, prefix, X.hist, &X.launches); });
        if (rc != PP_OK) return rc;
        uint32_t hist[512] = {};
        for (FilterSide& X : S) for (int i = 0; i < 512; ++i) hist[i] += X.hist[i];
        for (int r = 0; r < 2; ++r) prefix[r] |= filter_pick_digit(hist + r * 256, rank[r]) << shift;
        done_mask |= 255u << shift;
    }
    res->low = in_range[0] ? prefix[0] : 0;
    res->high = in_range[1] ? prefix[1] : 0;

    // ---- verdicts on the owners, then home to the sources
    rc = fx_all(S, [&](FilterSide& X, int) -> int {
        pp_ctx* ctx = X.ctx;
        cudaStream_t s = ctx->stream;
        filter_pass(ctx, X.f, res->low, res->high, (uint32_t)chosen, &X.launches);
        CK(cudaMemcpyAsync(X.np, X.f.n_pass, 16, cudaMemcpyDeviceToHost, s));
        CK(cudaStreamSynchronize(s));
        CK(cudaGetLastError());
        return PP_OK;
    });
    if (rc != PP_OK) return rc;
    rc = fx_all(S, [&](FilterSide& D, int d) -> int {
        for (uint32_t gg = 0; gg < n; ++gg) {
            const uint32_t g = ((uint32_t)d + gg) % n;
            FilterSide& X = S[g];
            for (int k = 0; k < 2; ++k) {
                const int r = fx_copy(D.ctx, X.ctx, X.ret + X.plan[(uint32_t)d].stage_rec[k], D.f.m[k].pass + rec_base(g, (uint32_t)d, k),
                                      X.cnt[(uint32_t)d].recs[k]);
                if (r != PP_OK) return r;
            }
        }
        pp_ctx* ctx = D.ctx;
        CK(cudaStreamSynchronize(ctx->stream));
        return PP_OK;
    });
    if (rc != PP_OK) return rc;
    return fx_all(S, [&](FilterSide& X, int) -> int {
        pp_ctx* ctx = X.ctx;
        const uint64_t st_recs = X.st_recs[0] + X.st_recs[1];
        if (st_recs) { k_fx_home<<<fx_blocks(st_recs, 256), 256, 0, ctx->stream>>>(X.s_recs, st_recs, X.ret, X.pass[0], X.pass[1]); X.launches++; }
        CK(cudaStreamSynchronize(ctx->stream));
        CK(cudaGetLastError());
        return PP_OK;
    });
}

// Writes one output file from its pieces, S[g].out_n bytes in context g's B->out, one after the other.  A regular file gets its final
// size up front and every piece is written at its offset, in parallel (a shared mapping or pwrite(); one thread per piece after the
// first).  Anything else - a FIFO, >(gzip ...), /dev/stdout into a pipe, /dev/null - cannot be truncated or written at offsets: the
// pieces are streamed in order with write(), like the reference's BufWriter (filter.rs:296-349).  Errors are reported on S[0]'s context.
static int write_pieces(const std::vector<FilterSide>& S, const char* path, uint64_t* out_bytes) {
    pp_ctx* c0 = S[0].ctx;
    const size_t n = S.size();
    std::vector<uint64_t> base(n + 1, 0);
    for (size_t g = 0; g < n; ++g) base[g + 1] = base[g] + S[g].out_n;
    const uint64_t out_n = base[n];
    struct stat osb;
    const bool special = stat(path, &osb) == 0 && !S_ISREG(osb.st_mode);
    const int ofd = special ? open(path, O_WRONLY) : open(path, O_RDWR | O_CREAT | O_TRUNC, 0666);
    if (ofd < 0) return c0->fail(PP_ERR_IO, std::string("unable to write alignments to \"") + path + "\"");
    std::vector<int> wrc(n, PP_OK), cuda_err(n, 0);
    bool stream_out = special;
    if (out_n && !stream_out && ftruncate(ofd, (off_t)out_n) != 0) stream_out = true;
    if (out_n && stream_out) {
        for (size_t g = 0; g < n && wrc[0] == PP_OK; ++g)
            if (S[g].out_n) wrc[0] = download_stream(S[g].ctx->device, S[g].T, S[g].B->out.as<uint8_t>(), ofd, S[g].out_n, &cuda_err[0]);
    } else if (out_n) {
        // Stores into a mapping cannot report "no space left" (they raise SIGBUS), so the mapping is only used when the file system has
        // room to spare; otherwise pwrite() reports the error like the reference does (filter.rs:307-311).
        struct statvfs vfs;
        const bool roomy = fstatvfs(ofd, &vfs) == 0 && (uint64_t)vfs.f_bavail * (uint64_t)vfs.f_frsize > 2 * out_n + (64ull << 20);
        void* map = roomy ? mmap(nullptr, (size_t)out_n, PROT_READ | PROT_WRITE, MAP_SHARED, ofd, 0) : MAP_FAILED;
        if (map == MAP_FAILED) map = nullptr;
        auto put = [&](size_t g) {
            wrc[g] = download_file(S[g].ctx->device, S[g].T, S[g].B->out.as<uint8_t>(), ofd, (uint8_t*)map, S[g].out_n, &cuda_err[g], base[g]);
        };
        std::vector<std::thread> th;
        for (size_t g = 1; g < n; ++g)
            if (S[g].out_n) th.emplace_back(put, g);
        if (S[0].out_n) put(0);
        for (auto& t : th) t.join();
        if (map && munmap(map, (size_t)out_n) != 0 && wrc[0] == PP_OK) wrc[0] = PP_ERR_IO;
    }
    int w = PP_OK, ce = 0;
    for (size_t g = 0; g < n; ++g) if (wrc[g] != PP_OK && w == PP_OK) { w = wrc[g]; ce = cuda_err[g]; }
    if (close(ofd) != 0 && w == PP_OK) w = PP_ERR_IO;
    if (w == PP_ERR_IO) return c0->fail(PP_ERR_IO, std::string("unable to write alignments to \"") + path + "\"");
    if (w == PP_ERR_CUDA) return c0->fail_cuda((cudaError_t)ce, "filtered SAM download", __FILE__, __LINE__);
    *out_bytes = out_n;
    return PP_OK;
}

int pp_filter_files_device(pp_ctx* const* ctxs, int n_ctx, const char* in1, const char* in2, const char* out1, const char* out2,
                           const pp_filter_params* prm, const uint64_t* const cuts[2], pp_filter_result* res, pp_filter_file_stats* fs,
                           pp_fused_polish* fuse) {
    const uint32_t n = (uint32_t)n_ctx;
    pp_ctx* c0 = ctxs[0];
    const char* ins[2] = {in1, in2};
    const char* outs[2] = {out1, out2};
    memset(fs, 0, sizeof *fs);
    const auto t_begin = std::chrono::steady_clock::now();
    auto t_mark = t_begin;
    auto lap = [&](int i) { const auto now = std::chrono::steady_clock::now(); fs->phase_ms[i] += std::chrono::duration<float, std::milli>(now - t_mark).count(); t_mark = now; };
    std::vector<FilterSide> S(n);
    for (uint32_t g = 0; g < n; ++g) {
        pp_ctx* ctx = ctxs[g];
        S[g].ctx = ctx;
        CK(cudaSetDevice(ctx->device));
        int rc = tok_state(ctx, &S[g].T);
        if (rc) { if (g) c0->err = ctx->err; return rc; }
        if (!S[g].T->fbufs) S[g].T->fbufs = new TokFilterBufs();
        S[g].B = S[g].T->fbufs;
        enable_peers(ctx, ctxs, n);
    }

    // ---- every context: its two texts into HBM, lines, quick parse
    int rc = fx_all(S, [&](FilterSide& X, int g) { return fx_text_in(X, g, ins, cuts); });
    if (rc != PP_OK) return rc;
    uint64_t n_al[2] = {0, 0};
    for (FilterSide& X : S) for (int k = 0; k < 2; ++k) { n_al[k] += X.n_al[k]; fs->text_bytes[k] += X.fd[k].n; }
    for (int k = 0; k < 2; ++k) fs->alignments[k] = n_al[k];
    if (n_al[0] == 0 || n_al[1] == 0) return PP_TOK_HOST;               // "no alignments found in ..." is worded by the host path
    if (n_al[0] >= 0x7FFFFFFFull || n_al[1] >= 0x7FFFFFFFull) return PP_TOK_HOST;

    // ---- the filter: one context on its own, several across the contexts by read name
    if (n == 1) {
        lap(0);                                                          // (over several contexts phase 0 also takes the local interning)
        rc = filter_one(S[0], prm, res, fuse != nullptr, lap);
    } else {
        rc = filter_exchange(S, prm, res, lap);
    }
    if (rc != PP_OK) return rc;
    uint64_t np[2] = {0, 0};
    for (FilterSide& X : S) { np[0] += X.np[0]; np[1] += X.np[1]; }
    res->n_pass = np[0] + np[1];
    for (int k = 0; k < 2; ++k) { fs->pass[k] = np[k]; fs->fail[k] = n_al[k] - np[k]; }
    lap(2);

    // ---- output text, file by file: every context assembles its piece (lengths -> offsets -> bytes), one writer puts the pieces in the file
    for (int k = 0; k < 2; ++k) {
        if (!outs[k]) continue;
        rc = fx_all(S, [&](FilterSide& X, int g) -> int {
            pp_ctx* ctx = X.ctx;
            TokState* T = X.T;
            TokFilterBufs& B = *X.B;
            cudaStream_t s = ctx->stream;
            const FileDev& fd = X.fd[k];
            const uint64_t nl = fd.n_lines;
            X.out_n = 0;
            if (!nl) return PP_OK;
            CK(B.table.ensure((nl + 2) * 8));                                // the local intern table is done with: reuse it
            unsigned long long* out_off = B.table.as<unsigned long long>();
            k_ftok_outlen<<<fx_blocks(nl + 1, TK_LINE_THREADS), TK_LINE_THREADS, 0, s>>>(fd, X.pass[k], out_off);
            size_t cub_bytes = 0;
            CK(cub::DeviceScan::ExclusiveSum(nullptr, cub_bytes, out_off, out_off, (int64_t)(nl + 1)));
            CK(T->cub.ensure(cub_bytes + 256));
            size_t tbb = T->cub.cap;
            CK(cub::DeviceScan::ExclusiveSum(T->cub.p, tbb, out_off, out_off, (int64_t)(nl + 1), s));
            CK(cudaMemcpyAsync(T->h_tot, out_off + nl, 8, cudaMemcpyDeviceToHost, s));
            CK(cudaStreamSynchronize(s));
            X.out_n = T->h_tot[0];
            if (g == 0) lap(3);                                              // (context 0 runs on the calling thread)
            TRY_ALLOC(B.out.ensure(X.out_n + 64));
            k_ftok_copy<<<fx_blocks(nl * 32, 256), 256, 0, s>>>(fd, X.pass[k], out_off, B.out.as<uint8_t>());
            CK(cudaStreamSynchronize(s));
            CK(cudaGetLastError());
            X.launches += n == 1 ? 4 : 3;                                    // (the N-context count takes the scan as one launch)
            if (g == 0) lap(4);
            return PP_OK;
        });
        if (rc != PP_OK) return rc;
        const auto t0 = std::chrono::steady_clock::now();
        rc = write_pieces(S, outs[k], &fs->out_bytes[k]);
        fs->d2h_ms += std::chrono::duration<float, std::milli>(std::chrono::steady_clock::now() - t0).count();
        if (rc != PP_OK) return rc;
        lap(5);
    }
    for (FilterSide& X : S) { fs->launches += X.launches; fs->h2d_ms = std::max(fs->h2d_ms, X.h2d_ms); }

    // ---- filter-polish: every context tokenises its text for polish (pp_tok_*), with its verdicts as ZP flags; byte ranges get the
    // range marks and the empty-range rule of pp_tok_add_files
    if (fuse) {
        fuse->rc = PP_TOK_HOST;
        for (int bits = 4;; bits = 8) {
            rc = fx_all(S, [&](FilterSide& X, int g) -> int {
                pp_ctx* ctx = X.ctx;
                TokState* T = X.T;
                int r = pp_tok_begin(ctx, fuse->fasta, fuse->careful, bits);
                if (r == PP_OK && cuts) {
                    const uint64_t off[2] = {cuts[0][g], cuts[1][g]}, len[2] = {cuts[0][g + 1] - cuts[0][g], cuts[1][g + 1] - cuts[1][g]};
                    r = pp_tok_set_ranges(ctx, off, len, 2);
                }
                if (r != PP_OK) return r;
                T->expect_total = X.fd[0].n + X.fd[1].n;
                memset(X.tst, 0, sizeof X.tst);
                for (int k = 0; k < 2; ++k) {
                    if (cuts) T->marks.push_back({T->aln_base, T->ops_base, T->blk_base, T->read_base});
                    const uint64_t a0 = T->aln_base;
                    r = tok_process(ctx, T, X.fd[k].text, X.fd[k].n, X.fd[k].unterminated != 0, &X.tst[k], cuts != nullptr);
                    if (r == PP_OK && X.tst[k].alignments != X.n_al[k]) r = PP_TOK_HOST;       // (cannot happen: same lines, same rule)
                    if (r != PP_OK) { T->active = false; return r; }
                    if (X.n_al[k]) {
                        k_apply_pass<<<fx_blocks(X.n_al[k], 256), 256, 0, ctx->stream>>>(ctx->b[B_FLAGS].as<uint8_t>() + a0, X.pass[k], X.n_al[k]);
                        CK(cudaStreamSynchronize(ctx->stream));
                        CK(cudaGetLastError());
                    }
                }
                if (cuts) T->marks.push_back({T->aln_base, T->ops_base, T->blk_base, T->read_base});
                return PP_OK;
            });
            if (rc == PP_TOK_NEED8 && bits == 4) continue;
            break;
        }
        if (rc == PP_TOK_NEED8) rc = PP_TOK_HOST;
        if (rc < 0) return rc;
        if (rc == PP_OK) {
            memset(fuse->stats, 0, sizeof fuse->stats);
            for (FilterSide& X : S)
                for (int k = 0; k < 2; ++k) {
                    fuse->stats[k].alignments += X.tst[k].alignments; fuse->stats[k].reads += X.tst[k].reads; fuse->stats[k].lines += X.tst[k].lines;
                }
            fuse->n_aln = n_al[0] + n_al[1];
        }
        fuse->rc = rc;
    }
    fs->total_ms = std::chrono::duration<float, std::milli>(std::chrono::steady_clock::now() - t_begin).count();
    return PP_OK;
}
