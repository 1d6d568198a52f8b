// pp_ctx.cuh — the device context shared by the CUDA translation units of libpolypolish_b200 (not part of the ABI).
#pragma once
#include <cuda_runtime.h>

#include <string>

#include "pp_internal.h"

struct DevStatus;
struct DevParams;
struct TokState;     // tok_kernels.cu
struct pp_ctx;
void pp_tok_release(pp_ctx* ctx);

struct DevBuf {
    void* p = nullptr;
    size_t cap = 0;
    cudaError_t ensure(size_t bytes) {
        if (bytes <= cap) return cudaSuccess;
        if (p) cudaFree(p);
        p = nullptr; cap = 0;
        size_t want = bytes + bytes / 8 + 256;
        cudaError_t e = cudaMalloc(&p, want);
        if (e == cudaSuccess) cap = want;
        return e;
    }
    void release() { if (p) cudaFree(p); p = nullptr; cap = 0; }
    template <class T> T* as() const { return (T*)p; }
};

enum { B_CONTIG, B_REFSTART, B_READID, B_SEQOFF, B_SEQLEN, B_CIGOFF, B_NCIG, B_NM, B_FLAGS, B_CIGOPS, B_SEQPOOL,
       B_DRAFT, B_CTGOFF, B_ZEROPOOL, B_RECS, B_KEY, B_VAL, B_SKEY, B_SVAL, B_BINSTART, B_SREC, B_SSEQ, B_KF, B_NK, B_TILEORDER, B_ERRC, B_GQ, B_HEADS, B_NODES, B_CUBTMP, B_SEQ2, B_OUT,
       B_OUTOFF, B_DEBUG, B_RES, B_RECAT, B_CHUNKDELTA, B_PARAMS, B_SCRATCH, B_SCRATCH2,
       B_CHG, B_CHGPOS, B_STRPOS, B_STRPOOL, B_STROFF, B_STS, B_RUNFIRST, B_RUNSTART, B_RUNSTS,
       B_DEPSTART, B_DEPRUN,
       B_TOKLINE, B_TOKTMP, B_TOKNAMES, B_COUNT };

// The resident dataset: DS_N arrays, array k in b[B_CONTIG + k].  Each is sized by one count - records, CIGAR ops or sequence blocks -
// times its element width; the sequence pool's width is the block bytes of the dataset's seq_bits.
enum DsCount { DS_RECS, DS_OPS, DS_BLKS };
struct DsArray { uint32_t width; DsCount count; };          // width 0: the sequence pool
enum { DS_SEQPOOL = B_SEQPOOL - B_CONTIG, DS_N };
constexpr DsArray DS_ARRAYS[DS_N] = {
    {4, DS_RECS},   // B_CONTIG    contig
    {4, DS_RECS},   // B_REFSTART  ref_start
    {4, DS_RECS},   // B_READID    read_id
    {4, DS_RECS},   // B_SEQOFF    seq_off
    {2, DS_RECS},   // B_SEQLEN    seq_len
    {4, DS_RECS},   // B_CIGOFF    cigar_off
    {2, DS_RECS},   // B_NCIG      n_cigar
    {4, DS_RECS},   // B_NM        nm
    {1, DS_RECS},   // B_FLAGS     flags
    {4, DS_OPS},    // B_CIGOPS    cigar_ops
    {0, DS_BLKS},   // B_SEQPOOL   seq_pool
};
__host__ __device__ constexpr uint32_t ds_block_bytes(uint32_t seq_bits) { return seq_bits == 8 ? 32 : 16; }
inline size_t ds_width(int k, uint32_t seq_bits) { return DS_ARRAYS[k].width ? DS_ARRAYS[k].width : ds_block_bytes(seq_bits); }
// bytes of array k for n[DS_RECS] records, n[DS_OPS] CIGAR ops and n[DS_BLKS] sequence blocks
inline size_t ds_bytes(int k, const uint64_t n[3], uint32_t seq_bits) { return (size_t)n[DS_ARRAYS[k].count] * ds_width(k, seq_bits); }

// The typed device pointers of one set of the DS_N arrays (a context's dataset, or a copy of its layout).
struct DsArrays {
    uint32_t *contig, *ref_start, *read_id, *seq_off;
    uint16_t* seq_len;
    uint32_t* cigar_off;
    uint16_t* n_cigar;
    uint32_t* nm;
    uint8_t* flags;
    uint32_t* cigar_ops;
    uint8_t* seq_pool;
};
inline DsArrays ds_view(const DevBuf* b) {                  // b[0 .. DS_N - 1] in the order above: ctx->b + B_CONTIG, or a copy's
    return {b[0].as<uint32_t>(), b[1].as<uint32_t>(), b[2].as<uint32_t>(), b[3].as<uint32_t>(), b[4].as<uint16_t>(), b[5].as<uint32_t>(),
            b[6].as<uint16_t>(), b[7].as<uint32_t>(), b[8].as<uint8_t>(), b[9].as<uint32_t>(), b[10].as<uint8_t>()};
}

// The host arrays of `a`, in the order above.
inline void ds_host(const pp_alignments* a, const void* out[DS_N]) {
    const void* p[DS_N] = {a->contig, a->ref_start, a->read_id, a->seq_off, a->seq_len, a->cigar_off, a->n_cigar, a->nm, a->flags,
                           a->cigar_ops, a->seq_pool};
    for (int k = 0; k < DS_N; ++k) out[k] = p[k];
}

// A per-position report recorded as runs: whether calls record it (on), whether the last call did (have) and its runs, exactly n
// long, in b[b_start] (start positions) / b[b_value] (values).
struct RunReport {
    bool on, have;
    uint32_t n;
    int b_start, b_value;
};

// The report files of the file-level commands that are set per context (pp_set_changes_file, pp_set_status_file, pp_set_vcf_file,
// pp_set_depth_file), in the order they are created after --debug's.
enum { F_CHANGES, F_STATUS, F_VCF, F_DEPTH, F_COUNT };

struct pp_ctx {
    int device = 0;
    cudaStream_t stream = nullptr;
    cudaStream_t copy_stream = nullptr;   // pp_dataset_upload: the sequence pool crosses PCIe while the records are binned
    cudaEvent_t ev_small = nullptr, ev_seq = nullptr;
    std::string err;
    DevBuf b[B_COUNT];
    cudaEvent_t ev[PP_N_STAGES + 4] = {};
    DevStatus* h_status = nullptr;        // pinned
    DevParams* h_params = nullptr;        // pinned
    uint8_t* h_init = nullptr;            // pinned image of the per-call reset block (run_polish)
    bool have_ds = false;
    // dataset facts
    uint64_t n_aln = 0, n_reads = 0, n_ops = 0, seq_bytes = 0, G = 0;
    uint32_t n_contigs = 0, seq_bits = 4;
    int sm_count = 132;
    uint32_t launches = 0;
    // sizes that adapt when a call overflows them (kept across calls on the same dataset)
    uint32_t node_cap = 0;
    uint32_t n_slots = 0, max_ext = 0;    // the binned dataset: alignments that can contribute, largest binned extent
    bool tile_attr_set = false;           // k_tile's dynamic shared memory opt-in done
    uint64_t out_cap = 0;
    bool global_k = false;
    bool debug_on = false, have_debug = false;
    const uint32_t* last_head = nullptr;
    uint32_t last_nodes = 0;
    // --changes (pp_polish_set_changes): the change list of the last call, its first capacity grows like node_cap
    bool changes_on = false, have_changes = false;
    uint32_t chg_cap = 0, n_changes = 0;
    int64_t chg_pool = -1;                // bytes of the change rows' allele strings in B_STRPOOL, -1 = not made yet
    // --status-bed (pp_polish_set_status) and --depth-bedgraph (pp_polish_set_depth): each one's runs of the last call
    RunReport status{false, false, 0, B_RUNSTART, B_RUNSTS}, depth{false, false, 0, B_DEPSTART, B_DEPRUN};
    std::string report_path[F_COUNT];     // pp_set_*_file: the reports the file-level commands also write ("" = none)
    TokState* tok = nullptr;              // SAM tokeniser state (tok_kernels.cu), created on first use
    int parser = 0;                       // pp_set_parser: 0 device tokeniser where possible, 1 host packer only
    std::string* log = nullptr;           // pp_batch_files: the running job's verbose log goes here instead of stderr (pp_log)

    int fail(int code, const std::string& m) { err = m; return code; }
    int fail_cuda(cudaError_t e, const char* what, const char* file, int line) {
        const char* base = file;
        for (const char* q = file; *q; ++q) if (*q == '/') base = q + 1;
        err = std::string("CUDA error: ") + cudaGetErrorString(e) + " at " + what + " (" + base + ":" + std::to_string(line) + ")";
        return PP_ERR_CUDA;
    }
};

#define CK(x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) return ctx->fail_cuda(e_, #x, __FILE__, __LINE__); } while (0)
