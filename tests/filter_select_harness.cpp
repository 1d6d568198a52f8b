// CPU harness for the filter's insert-size select (polypolish_b200/csrc/filter_dev.h), compiled by tests/test_filter_select_cpu.py
// with g++.  It runs the rounds the way pp_filter_core and the multi-GPU path do: per round, the two histograms k_f_hist counts
// (filter_hist_rows under each rank's prefix), summed over `n_owners` owners as the host does for several GPUs, then filter_pick_digit.
#include <string.h>

#include "../polypolish_b200/csrc/filter_dev.h"

extern "C" {

unsigned long long h_nearest_rank(double percentile, unsigned long long n) { return nearest_rank(percentile, n); }

// v[n]: the insert sizes of the chosen orientation; value i belongs to owner i % n_owners.  out[2] = low, high (0 where the rank is
// past the list, as pp_filter reports them).  trace[round][rank][3] = digit picked, rank inside its bucket, the bucket's count.
int h_select(const uint32_t* v, unsigned long long n, uint32_t n_owners, double low_pct, double high_pct, uint32_t* out, uint32_t* trace) {
    if (n_owners < 1 || n_owners > 64) return -1;
    pp_filter_params prm;
    memset(&prm, 0, sizeof prm);
    prm.low_pct = low_pct;
    prm.high_pct = high_pct;
    bool in_range[2];
    unsigned long long rank[2];
    filter_ranks(&prm, n, rank, in_range);
    uint32_t prefix[2] = {0, 0}, done_mask = 0;
    int round = 0;
    static uint32_t owner_hist[64][512];
    for (const int shift : FILTER_SHIFTS) {
        memset(owner_hist, 0, sizeof owner_hist);
        for (unsigned long long i = 0; i < n; ++i) {
            const uint32_t d = (v[i] >> shift) & 255u, rows = filter_hist_rows(v[i], done_mask, prefix[0], prefix[1]);
            if (rows & 1u) owner_hist[i % n_owners][d] += 1;
            if (rows & 2u) owner_hist[i % n_owners][256 + d] += 1;
        }
        uint32_t hist[512] = {};
        for (uint32_t o = 0; o < n_owners; ++o)
            for (int i = 0; i < 512; ++i) hist[i] += owner_hist[o][i];
        for (int r = 0; r < 2; ++r) {
            const uint32_t d = filter_pick_digit(hist + r * 256, rank[r]);
            prefix[r] |= d << shift;
            if (trace && round < 4) {
                trace[(round * 2 + r) * 3 + 0] = d;
                trace[(round * 2 + r) * 3 + 1] = (uint32_t)rank[r];
                trace[(round * 2 + r) * 3 + 2] = hist[r * 256 + d];
            }
        }
        done_mask |= 255u << shift;
        ++round;
    }
    out[0] = in_range[0] ? prefix[0] : 0;
    out[1] = in_range[1] ? prefix[1] : 0;
    return round;
}
}
