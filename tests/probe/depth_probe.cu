// depth_probe.cu — the depth helpers of polypolish_b200/csrc/polish_dev.cuh, one input element at a time: depth_deficit(k),
// depth_bounds(cover, deficit), bankers_rounding(x) and vote_thresholds(prm, x), so that tests/test_depth_bounds.py can check
// them against exact rational arithmetic.  Built twice by tests/probe_lib.py: for the CPU against tests/emu/cuda_emu.h (the
// emulated directed rounding), and for sm_90a with the product's nvcc flags (the hardware __dadd_ru, __ull2double_rd, ...).
// TEST INFRASTRUCTURE: nothing in polypolish_b200/ links or loads this.
#ifdef PROBE_CPU
#include "../emu/cuda_emu.h"
#else
#include <cuda_runtime.h>
#endif

#include "../../polypolish_b200/csrc/polish_dev.cuh"

struct ProbeIn {                     // (tests/probe_lib.py IN_DTYPE)
    uint32_t k, cover;
    unsigned long long deficit;
    double x, fv, fi;
    uint32_t min_depth, pad;
};
struct ProbeOut {                    // (tests/probe_lib.py OUT_DTYPE)
    unsigned long long dd;
    double lo, hi, fx;
    uint32_t br, vt, it, low;
};

__device__ __forceinline__ void probe_one(const ProbeIn& in, ProbeOut& out) {
    out.dd = in.k >= 2 ? depth_deficit(in.k) : 0ull;
    const DepthBounds b = depth_bounds(in.cover, in.deficit);
    out.lo = b.lo; out.hi = b.hi; out.fx = b.fx;
    out.br = bankers_rounding(in.x);
    DevParams prm;
    prm.fv = in.fv; prm.fi = in.fi; prm.min_depth = in.min_depth; prm.max_errors = 0; prm.careful = 0; prm.pad = 0;
    const Thresholds t = vote_thresholds(prm, in.x);
    out.vt = t.vt; out.it = t.it; out.low = t.low ? 1u : 0u;
}

#ifdef PROBE_CPU
extern "C" int depth_probe(const ProbeIn* in, ProbeOut* out, unsigned long long n) {
    for (unsigned long long i = 0; i < n; ++i) probe_one(in[i], out[i]);
    return 0;
}
#else
__global__ void k_depth_probe(const ProbeIn* in, ProbeOut* out, unsigned long long n) {
    const unsigned long long i = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) probe_one(in[i], out[i]);
}

// One thread per element on the current device; returns the first CUDA error (0 = cudaSuccess).  Frees what it allocated on
// every path.
extern "C" int depth_probe(const ProbeIn* in, ProbeOut* out, unsigned long long n) {
    if (n == 0) return 0;
    ProbeIn* d_in = nullptr;
    ProbeOut* d_out = nullptr;
    cudaError_t e = cudaMalloc(&d_in, n * sizeof(ProbeIn));
    if (e == cudaSuccess) e = cudaMalloc(&d_out, n * sizeof(ProbeOut));
    if (e == cudaSuccess) e = cudaMemcpy(d_in, in, n * sizeof(ProbeIn), cudaMemcpyHostToDevice);
    if (e == cudaSuccess) {
        k_depth_probe<<<(unsigned)((n + 255) / 256), 256>>>(d_in, d_out, n);
        e = cudaGetLastError();
    }
    if (e == cudaSuccess) e = cudaDeviceSynchronize();
    if (e == cudaSuccess) e = cudaMemcpy(out, d_out, n * sizeof(ProbeOut), cudaMemcpyDeviceToHost);
    const cudaError_t f1 = d_in ? cudaFree(d_in) : cudaSuccess, f2 = d_out ? cudaFree(d_out) : cudaSuccess;
    if (e == cudaSuccess) e = f1 != cudaSuccess ? f1 : f2;
    return (int)e;
}
#endif
