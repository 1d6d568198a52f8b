// filter_kernels.cu — `polypolish filter` on the device: insert-size thresholds + per-alignment pair QC.
//
// Replaces (reference = Polypolish src/filter.rs):
//   load_alignments' name-keyed grouping     :91-145   -> k_f_build   (per-name counts + linked lists)
//   get_insert_size_thresholds               :148-186  -> k_f_pairs   (unique pairs: orientation, insert size)
//   get_orientation / get_insert_size        :189-218  -> orient_insert()
//   sort_unstable + get_percentile           :178-180,249-259 -> k_f_hist / k_f_pick (exact radix select,
//                                               nearest-rank; the rank arithmetic stays in IEEE double on the host)
//   alignment_pass_qc                        :352-377  -> k_f_pass
// Integer work only; ~18 B per record.  The reference's HashMap<String, Vec<Alignment>> becomes two dense arrays per
// mate indexed by the QNAME id the host assigns (count, list head) plus a per-record `next` link, so "does ANY
// alignment of the mate make a good pair" is a short list walk.
#include <cuda_runtime.h>

#include <algorithm>
#include <cmath>
#include <string>
#include <vector>

#include "pp_internal.h"

// context pieces shared with polish_kernels.cu
int pp_ctx_device(pp_ctx* ctx);
int pp_ctx_sm_count(pp_ctx* ctx);
cudaStream_t pp_ctx_stream(pp_ctx* ctx);
int pp_ctx_fail_cuda(pp_ctx* ctx, cudaError_t e, const char* what, const char* file, int line);
void* pp_ctx_scratch(pp_ctx* ctx, size_t bytes);       // grows a ctx-owned device buffer; nullptr on failure
void pp_ctx_count_launches(pp_ctx* ctx, uint32_t n);
cudaEvent_t pp_ctx_event(pp_ctx* ctx, int i);

#define CKF(x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) return pp_ctx_fail_cuda(ctx, e_, #x, "filter_kernels.cu", __LINE__); } while (0)

#include "filter_dev.h"

// filter.rs:189-218.  Orientation codes: 0 fr, 1 rf, 2 ff, 3 rr.
__device__ __forceinline__ void orient_insert(uint32_t s1, uint32_t e1, bool rev1, uint32_t s2, uint32_t e2, bool rev2,
                                              uint32_t& orientation, uint32_t& insert) {
    const uint32_t p1 = rev1 ? e1 : s1, p2 = rev2 ? e2 : s2;
    if (rev1 != rev2) {
        // strands (s1, s2); the string is s1s2 when p1 < p2, else s2s1
        const bool first_is_f = (p1 < p2) ? !rev1 : !rev2;
        orientation = first_is_f ? 0u : 1u;
    } else if (!rev1) {
        orientation = (p1 < p2) ? 2u : 3u;
    } else {
        orientation = (p2 < p1) ? 2u : 3u;
    }
    const uint32_t lo = min(min(s1, e1), min(s2, e2)), hi = max(max(s1, e1), max(s2, e2));
    insert = hi - lo;
}

__global__ void __launch_bounds__(256) k_f_build(FilterDev f, int which) {
    const Mate& m = f.m[which];
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < m.n; i += gridDim.x * blockDim.x) {
        const uint32_t id = m.name_id[i];
        atomicAdd(&m.cnt[id], 1u);
        m.next[i] = atomicExch(&m.head[id], i);
    }
}

__global__ void __launch_bounds__(256) k_f_pairs(FilterDev f) {
    __shared__ unsigned long long s_pairs[4];
    if (threadIdx.x < 4) s_pairs[threadIdx.x] = 0;
    __syncthreads();
    for (uint32_t id = blockIdx.x * blockDim.x + threadIdx.x; id < f.n_names; id += gridDim.x * blockDim.x) {
        uint8_t o = 255;
        if (f.m[0].cnt[id] == 1 && f.m[1].cnt[id] == 1) {           // filter.rs:156-161
            const uint32_t a = f.m[0].head[id], b = f.m[1].head[id];
            if (f.m[0].contig[a] == f.m[1].contig[b]) {
                uint32_t orientation, insert;
                orient_insert(f.m[0].ref_start[a], f.m[0].ref_end[a], f.m[0].flags[a] & 1, f.m[1].ref_start[b], f.m[1].ref_end[b],
                              f.m[1].flags[b] & 1, orientation, insert);
                o = (uint8_t)orientation;
                f.ins[id] = insert;
                atomicAdd(&s_pairs[orientation], 1ull);
            }
        }
        f.ori[id] = o;
    }
    __syncthreads();
    if (threadIdx.x < 4 && s_pairs[threadIdx.x]) atomicAdd(&f.pairs[threadIdx.x], s_pairs[threadIdx.x]);
}

// One 8-bit digit of an exact radix select over { ins[id] : ori[id] == chosen }, for two ranks at once.
__global__ void __launch_bounds__(256) k_f_hist(FilterDev f, uint32_t chosen, int shift, uint32_t done_mask) {
    __shared__ uint32_t s_h[2][256];
    s_h[0][threadIdx.x] = 0;
    s_h[1][threadIdx.x] = 0;
    __syncthreads();
    const uint32_t p0 = f.sel_prefix[0], p1 = f.sel_prefix[1];
    for (uint32_t id = blockIdx.x * blockDim.x + threadIdx.x; id < f.n_names; id += gridDim.x * blockDim.x) {
        if (f.ori[id] != chosen) continue;
        const uint32_t v = f.ins[id], d = (v >> shift) & 255u, rows = filter_hist_rows(v, done_mask, p0, p1);
        if (rows & 1u) atomicAdd(&s_h[0][d], 1u);
        if (rows & 2u) atomicAdd(&s_h[1][d], 1u);
    }
    __syncthreads();
    if (s_h[0][threadIdx.x]) atomicAdd(&f.hist[threadIdx.x], s_h[0][threadIdx.x]);
    if (s_h[1][threadIdx.x]) atomicAdd(&f.hist[256 + threadIdx.x], s_h[1][threadIdx.x]);
}

__global__ void k_f_pick(FilterDev f, int shift) {      // one warp; lanes 0 and 1 pick the digit of rank 0 / 1
    const int r = threadIdx.x;
    if (r < 2) {
        unsigned long long rank = f.sel_rank[r];
        f.sel_prefix[r] |= filter_pick_digit(f.hist + r * 256, rank) << shift;
        f.sel_rank[r] = rank;
    }
    __syncthreads();
    for (int i = r; i < 512; i += 32) f.hist[i] = 0;
}

__global__ void __launch_bounds__(256) k_f_pass(FilterDev f, int which, uint32_t low, uint32_t high, uint32_t chosen) {
    const Mate& me = f.m[which];
    const Mate& mate = f.m[1 - which];
    unsigned long long npass = 0;
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < me.n; i += gridDim.x * blockDim.x) {
        const uint32_t id = me.name_id[i];
        bool pass = mate.cnt[id] == 0 || me.cnt[id] == 1;           // filter.rs:362-367
        if (!pass) {
            const uint32_t c = me.contig[i], s = me.ref_start[i], e = me.ref_end[i];
            const bool rev = me.flags[i] & 1;
            for (uint32_t j = mate.head[id]; j != 0xFFFFFFFFu && !pass; j = mate.next[j]) {
                uint32_t orientation, insert;
                // get_insert_size(a, pair) and get_orientation(a, pair): `a` is always the first argument
                orient_insert(s, e, rev, mate.ref_start[j], mate.ref_end[j], mate.flags[j] & 1, orientation, insert);
                pass = mate.contig[j] == c && low <= insert && insert <= high && orientation == chosen;
            }
        }
        me.pass[i] = pass ? 1 : 0;
        npass += pass;
    }
    for (int o = 16; o > 0; o >>= 1) npass += __shfl_down_sync(0xffffffffu, npass, o);
    if ((threadIdx.x & 31) == 0 && npass) atomicAdd(f.n_pass + which, npass);
}

static unsigned grid_for(pp_ctx* ctx, size_t n) {
    return (unsigned)std::min<size_t>(std::max<size_t>((n + 255) / 256, 1), (size_t)pp_ctx_sm_count(ctx) * 8);
}

int filter_begin(pp_ctx* ctx, const Mate in[2], uint32_t nn, FilterDev* out, uint32_t* launches) {
    cudaStream_t s = pp_ctx_stream(ctx);
    size_t off = 0;
    auto carve = [&](size_t bytes) { size_t o = off; off += (bytes + 255) & ~size_t(255); return o; };
    size_t o_cnt[2], o_head[2], o_next[2], o_pass[2];
    for (int k = 0; k < 2; ++k) { o_next[k] = carve((size_t)in[k].n * 4); o_pass[k] = carve((size_t)in[k].n + 1); }
    const size_t zero_begin = off;                       // zero-initialised block
    for (int k = 0; k < 2; ++k) o_cnt[k] = carve((size_t)nn * 4);
    const size_t o_pairs = carve(32), o_hist = carve(512 * 4), o_selp = carve(8), o_selr = carve(16), o_np = carve(16);
    const size_t zero_end = off;
    for (int k = 0; k < 2; ++k) o_head[k] = carve((size_t)nn * 4);   // 0xFF-initialised block
    const size_t ff_end = off;
    const size_t o_ins = carve((size_t)nn * 4), o_ori = carve(nn);
    uint8_t* base = (uint8_t*)pp_ctx_scratch(ctx, off + 256);
    if (!base) return pp_ctx_fail(ctx, PP_ERR_NOMEM, "pp_filter: device allocation failed");

    FilterDev& f = *out;
    for (int k = 0; k < 2; ++k) {
        f.m[k] = in[k];
        f.m[k].cnt = (uint32_t*)(base + o_cnt[k]); f.m[k].head = (uint32_t*)(base + o_head[k]);
        f.m[k].next = (uint32_t*)(base + o_next[k]); f.m[k].pass = base + o_pass[k];
    }
    f.n_names = nn;
    f.ins = (uint32_t*)(base + o_ins); f.ori = base + o_ori;
    f.pairs = (unsigned long long*)(base + o_pairs); f.hist = (uint32_t*)(base + o_hist);
    f.sel_prefix = (uint32_t*)(base + o_selp); f.sel_rank = (unsigned long long*)(base + o_selr);
    f.n_pass = (unsigned long long*)(base + o_np);
    CKF(cudaMemsetAsync(base + zero_begin, 0, zero_end - zero_begin, s));
    CKF(cudaMemsetAsync(base + zero_end, 0xFF, ff_end - zero_end, s));
    CKF(cudaEventRecord(pp_ctx_event(ctx, 1), s));
    for (int k = 0; k < 2; ++k)
        if (in[k].n) { k_f_build<<<grid_for(ctx, in[k].n), 256, 0, s>>>(f, k); ++*launches; }
    k_f_pairs<<<grid_for(ctx, nn), 256, 0, s>>>(f);
    ++*launches;
    return PP_OK;
}

int filter_orientation(pp_ctx* ctx, const pp_filter_params* prm, const unsigned long long pairs[4], int* chosen_out,
                       unsigned long long* n_sizes) {
    // filter.rs:168-177, 221-246
    if (pairs[0] + pairs[1] + pairs[2] + pairs[3] == 0)
        return pp_ctx_fail(ctx, PP_ERR_INPUT, "no one-alignment-per-read pairs available to determine orientation and insert size thresholds");
    int chosen = prm->orientation;
    if (chosen < 0) {
        unsigned long long mx = std::max(std::max(pairs[0], pairs[1]), std::max(pairs[2], pairs[3]));
        int n_max = 0;
        for (int i = 0; i < 4; ++i) if (pairs[i] == mx) { n_max++; chosen = i; }
        if (n_max != 1) return pp_ctx_fail(ctx, PP_ERR_INPUT, "could not automatically determine read pair orientation");
    }
    *n_sizes = (chosen >= 0 && chosen < 4) ? pairs[chosen] : 0;
    if (*n_sizes == 0) return pp_ctx_fail(ctx, PP_ERR_INPUT, "no read pairs available to determine insert size thresholds");
    *chosen_out = chosen;
    return PP_OK;
}

int filter_hist(pp_ctx* ctx, const FilterDev& f, uint32_t chosen, int shift, uint32_t done_mask, const uint32_t prefix[2], uint32_t hist[512],
                uint32_t* launches) {
    cudaStream_t s = pp_ctx_stream(ctx);
    CKF(cudaMemcpyAsync(f.sel_prefix, prefix, 8, cudaMemcpyHostToDevice, s));
    CKF(cudaMemsetAsync(f.hist, 0, 512 * 4, s));
    k_f_hist<<<grid_for(ctx, f.n_names), 256, 0, s>>>(f, chosen, shift, done_mask);
    ++*launches;
    CKF(cudaMemcpyAsync(hist, f.hist, 512 * 4, cudaMemcpyDeviceToHost, s));
    CKF(cudaStreamSynchronize(s));
    CKF(cudaGetLastError());
    return PP_OK;
}

void filter_pass(pp_ctx* ctx, const FilterDev& f, uint32_t low, uint32_t high, uint32_t chosen, uint32_t* launches) {
    for (int k = 0; k < 2; ++k)
        if (f.m[k].n) { k_f_pass<<<grid_for(ctx, f.m[k].n), 256, 0, pp_ctx_stream(ctx)>>>(f, k, low, high, chosen); ++*launches; }
}

// The filter proper on device-resident mate arrays (in[k].name_id / contig / ref_start / ref_end / flags and n set by the
// caller; host arrays are uploaded by pp_filter, the device SAM path of tok_kernels.cu builds them in place).
// res->pass1/pass2 may be null: the flags then stay on the device only (d_pass[k], inside the context's scratch buffer,
// valid until the next call that uses it).  n_pass_mate[k] = passing records of mate k.
int pp_filter_core(pp_ctx* ctx, const Mate in[2], const pp_filter_params* prm, pp_filter_result* res, const uint8_t* d_pass[2],
                   uint64_t n_pass_mate[2]) {
    cudaStream_t s = pp_ctx_stream(ctx);
    const uint32_t nn = (uint32_t)prm->n_names;
    FilterDev f;
    uint32_t launches = 0;
    int rc = filter_begin(ctx, in, nn, &f, &launches);
    if (rc != PP_OK) return rc;
    unsigned long long pairs[4];
    CKF(cudaMemcpyAsync(pairs, f.pairs, 32, cudaMemcpyDeviceToHost, s));
    CKF(cudaStreamSynchronize(s));
    CKF(cudaGetLastError());
    for (int i = 0; i < 4; ++i) res->pairs[i] = pairs[i];
    int chosen = 0;
    unsigned long long n_sizes = 0;
    rc = filter_orientation(ctx, prm, pairs, &chosen, &n_sizes);
    if (rc != PP_OK) return rc;
    res->orientation = chosen;

    // exact nearest-rank percentiles by radix select (two ranks at once)
    uint32_t thr[2] = {0, 0};
    bool in_range[2];
    unsigned long long sel_rank[2];
    filter_ranks(prm, n_sizes, sel_rank, in_range);
    CKF(cudaMemcpyAsync(f.sel_rank, sel_rank, 16, cudaMemcpyHostToDevice, s));
    uint32_t done_mask = 0;
    for (const int shift : FILTER_SHIFTS) {
        k_f_hist<<<grid_for(ctx, nn), 256, 0, s>>>(f, (uint32_t)chosen, shift, done_mask);
        k_f_pick<<<1, 32, 0, s>>>(f, shift);
        launches += 2;
        done_mask |= 255u << shift;
    }
    CKF(cudaMemcpyAsync(thr, f.sel_prefix, 8, cudaMemcpyDeviceToHost, s));
    CKF(cudaStreamSynchronize(s));
    CKF(cudaGetLastError());
    res->low = in_range[0] ? thr[0] : 0;
    res->high = in_range[1] ? thr[1] : 0;

    filter_pass(ctx, f, res->low, res->high, (uint32_t)chosen, &launches);
    CKF(cudaEventRecord(pp_ctx_event(ctx, 2), s));
    if (in[0].n && res->pass1) CKF(cudaMemcpyAsync(res->pass1, f.m[0].pass, in[0].n, cudaMemcpyDeviceToHost, s));
    if (in[1].n && res->pass2) CKF(cudaMemcpyAsync(res->pass2, f.m[1].pass, in[1].n, cudaMemcpyDeviceToHost, s));
    unsigned long long np[2] = {0, 0};
    CKF(cudaMemcpyAsync(np, f.n_pass, 16, cudaMemcpyDeviceToHost, s));
    CKF(cudaEventRecord(pp_ctx_event(ctx, 3), s));
    CKF(cudaStreamSynchronize(s));
    CKF(cudaGetLastError());
    res->n_pass = np[0] + np[1];
    if (n_pass_mate) { n_pass_mate[0] = np[0]; n_pass_mate[1] = np[1]; }
    if (d_pass) { d_pass[0] = f.m[0].pass; d_pass[1] = f.m[1].pass; }
    memset(&res->timing, 0, sizeof res->timing);
    float ms;
    CKF(cudaEventElapsedTime(&ms, pp_ctx_event(ctx, 0), pp_ctx_event(ctx, 1))); res->timing.stage_ms[6] = ms;
    CKF(cudaEventElapsedTime(&ms, pp_ctx_event(ctx, 1), pp_ctx_event(ctx, 2))); res->timing.stage_ms[1] = ms;
    CKF(cudaEventElapsedTime(&ms, pp_ctx_event(ctx, 2), pp_ctx_event(ctx, 3))); res->timing.stage_ms[7] = ms;
    CKF(cudaEventElapsedTime(&ms, pp_ctx_event(ctx, 0), pp_ctx_event(ctx, 3))); res->timing.total_ms = ms;
    res->timing.launches = launches;
    pp_ctx_count_launches(ctx, launches);
    return PP_OK;
}

void* pp_ctx_scratch2(pp_ctx* ctx, size_t bytes);      // a second ctx-owned device buffer (inputs of pp_filter)

extern "C" int pp_filter(pp_ctx* ctx, const pp_filter_mate* m1, const pp_filter_mate* m2, const pp_filter_params* prm,
                         pp_filter_result* res) {
    if (!ctx) return PP_ERR_ARG;
    if (!m1 || !m2 || !prm || !res) return pp_ctx_fail(ctx, PP_ERR_ARG, "pp_filter: null argument");
    if (m1->n >= 0xFFFFFFFFull || m2->n >= 0xFFFFFFFFull || prm->n_names >= 0xFFFFFFFFull)
        return pp_ctx_fail(ctx, PP_ERR_ARG, "pp_filter: more than 2^32-1 records or names");
    if ((m1->n && !res->pass1) || (m2->n && !res->pass2)) return pp_ctx_fail(ctx, PP_ERR_ARG, "pp_filter: null pass array");
    // filter.rs:47-52
    if (!(prm->low_pct > 0.0 && prm->low_pct < 50.0)) return pp_ctx_fail(ctx, PP_ERR_INPUT, "--low must be greater than 0 and less than 50");
    if (!(prm->high_pct > 50.0 && prm->high_pct < 100.0)) return pp_ctx_fail(ctx, PP_ERR_INPUT, "--high must be greater than 50 and less than 100");
    CKF(cudaSetDevice(pp_ctx_device(ctx)));
    cudaStream_t s = pp_ctx_stream(ctx);
    const pp_filter_mate* hm[2] = {m1, m2};
    size_t off = 0;
    auto carve = [&](size_t bytes) { size_t o = off; off += (bytes + 255) & ~size_t(255); return o; };
    size_t o_in[2][5];
    for (int k = 0; k < 2; ++k) {
        for (int a = 0; a < 4; ++a) o_in[k][a] = carve(hm[k]->n * 4);
        o_in[k][4] = carve(hm[k]->n);
    }
    uint8_t* base = (uint8_t*)pp_ctx_scratch2(ctx, off + 256);
    if (!base) return pp_ctx_fail(ctx, PP_ERR_NOMEM, "pp_filter: device allocation failed");
    CKF(cudaEventRecord(pp_ctx_event(ctx, 0), s));
    Mate in[2];
    for (int k = 0; k < 2; ++k) {
        const pp_filter_mate* h = hm[k];
        const void* src[5] = {h->name_id, h->contig, h->ref_start, h->ref_end, h->flags};
        for (int a = 0; a < 5; ++a)
            if (h->n) CKF(cudaMemcpyAsync(base + o_in[k][a], src[a], h->n * (a < 4 ? 4 : 1), cudaMemcpyHostToDevice, s));
        in[k].name_id = (const uint32_t*)(base + o_in[k][0]); in[k].contig = (const uint32_t*)(base + o_in[k][1]);
        in[k].ref_start = (const uint32_t*)(base + o_in[k][2]); in[k].ref_end = (const uint32_t*)(base + o_in[k][3]);
        in[k].flags = base + o_in[k][4];
        in[k].cnt = nullptr; in[k].head = nullptr; in[k].next = nullptr; in[k].pass = nullptr;
        in[k].n = (uint32_t)h->n;
    }
    return pp_filter_core(ctx, in, prm, res, nullptr, nullptr);
}
