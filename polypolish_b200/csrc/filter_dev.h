// filter_dev.h — the device-side interface of the filter proper (filter_kernels.cu), shared with the device SAM path
// (tok_kernels.cu).  Not part of the ABI.
#pragma once
#include <math.h>
#include <stdint.h>

#include "../../include/pp_abi.h"

struct Mate {
    const uint32_t *name_id, *contig, *ref_start, *ref_end;
    const uint8_t* flags;
    uint32_t* cnt;     // [n_names] aligned records per name
    uint32_t* head;    // [n_names] list head (record index) or 0xFFFFFFFF
    uint32_t* next;    // [n] next record of the same name
    uint8_t* pass;     // [n]
    uint32_t n;
};

struct FilterDev {
    Mate m[2];
    uint32_t n_names;
    uint32_t* ins;             // [n_names] insert size of the unique pair
    uint8_t* ori;              // [n_names] orientation 0..3 of the unique pair, 255 = not a unique pair
    unsigned long long* pairs; // [4]
    // radix select state for two ranks
    uint32_t* hist;            // [2][256]
    uint32_t* sel_prefix;      // [2]
    unsigned long long* sel_rank; // [2] remaining rank (1-based) inside the current prefix
    unsigned long long* n_pass;   // [2] passing records per mate
};

#ifdef __CUDACC__
#define FILTER_HD __host__ __device__
#else
#define FILTER_HD
#endif

// The radix select's rounds, most significant digit first.  The round at `shift` counts, for each rank, the values whose digits above
// `shift` equal that rank's prefix (done_mask covers them), by their digit at `shift`; the rank's digit is picked, and done_mask grows by it.
static constexpr int FILTER_SHIFTS[] = {24, 16, 8, 0};

// Which of the two histograms of a round value v counts in: bit r = rank r.
FILTER_HD inline uint32_t filter_hist_rows(uint32_t v, uint32_t done_mask, uint32_t prefix0, uint32_t prefix1) {
    return ((v & done_mask) == prefix0 ? 1u : 0u) | ((v & done_mask) == prefix1 ? 2u : 0u);
}

// One digit of the radix select: the bucket of `hist` (256 counts) that holds the rank-th value; `rank` becomes the rank inside it.
FILTER_HD inline uint32_t filter_pick_digit(const uint32_t* hist, unsigned long long& rank) {
    uint32_t d = 0;
    for (; d < 256; ++d) {
        const uint32_t c = hist[d];
        if (rank <= c) break;
        rank -= c;
    }
    return d > 255 ? 255 : d;
}

// filter.rs:249-259: rank = max(1, ceil(p / 100 * n) as usize)
inline unsigned long long nearest_rank(double percentile, unsigned long long n) {
    const double fraction = percentile / 100.0;
    const double r = ceil(fraction * (double)n);
    unsigned long long rank;
    if (!(r == r) || r <= 0.0) rank = 0;
    else if (r >= 18446744073709551615.0) rank = ~0ull;
    else rank = (unsigned long long)r;
    return rank < 1 ? 1 : rank;
}

// The two nearest ranks and whether each exists (sorted_list.get(rank - 1).unwrap_or(0)); a rank past the list selects rank 1, unused.
inline void filter_ranks(const pp_filter_params* prm, unsigned long long n_sizes, unsigned long long sel_rank[2], bool in_range[2]) {
    const unsigned long long ranks[2] = {nearest_rank(prm->low_pct, n_sizes), nearest_rank(prm->high_pct, n_sizes)};
    for (int r = 0; r < 2; ++r) {
        in_range[r] = ranks[r] <= n_sizes;
        sel_rank[r] = in_range[r] ? ranks[r] : 1;
    }
}

// The filter proper in phases (filter_kernels.cu), so that one context (pp_filter_core) and several (tok_kernels.cu, each holding
// the records of the read names it owns) run the same kernels and the same rules:
//   filter_begin        per-name lists and unique pairs (k_f_build, k_f_pairs); f->pairs is ready when the stream is
//   filter_orientation  the chosen orientation from the four pair counts, or the reference's error (filter.rs:168-177, 221-246)
//   filter_ranks        the two nearest ranks (filter.rs:249-259) and whether each exists (sorted_list.get(rank - 1).unwrap_or(0))
//   filter_hist         one digit of the radix select under the given prefixes: the 2 x 256 counts, on the host
//   filter_pass         alignment_pass_qc for every record (k_f_pass); f->m[k].pass and f->n_pass are ready when the stream is
int filter_begin(pp_ctx* ctx, const Mate in[2], uint32_t n_names, FilterDev* f, uint32_t* launches);
int filter_orientation(pp_ctx* ctx, const pp_filter_params* prm, const unsigned long long pairs[4], int* chosen, unsigned long long* n_sizes);
int filter_hist(pp_ctx* ctx, const FilterDev& f, uint32_t chosen, int shift, uint32_t done_mask, const uint32_t prefix[2], uint32_t hist[512],
                uint32_t* launches);
void filter_pass(pp_ctx* ctx, const FilterDev& f, uint32_t low, uint32_t high, uint32_t chosen, uint32_t* launches);

int pp_filter_core(pp_ctx* ctx, const Mate in[2], const pp_filter_params* prm, pp_filter_result* res, const uint8_t* d_pass[2],
                   uint64_t n_pass_mate[2]);
