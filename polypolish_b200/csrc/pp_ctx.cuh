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
