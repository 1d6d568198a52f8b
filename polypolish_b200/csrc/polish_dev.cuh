// polish_dev.cuh — the polish hot path as sm_90a device code.  Included by polish_kernels.cu (nvcc; host side, C ABI) and,
// for logic checks without a GPU, by tests/emu/emu_polish.cpp (g++ with tests/emu/cuda_emu.h standing in for CUDA).
//
// Replaces, on the device (reference = Polypolish v0.6.1, src/):
//   process_one_read            alignment.rs:275-305  -> k_goodk (goodness, k = #good per read group, --careful, unknown-contig /
//                                                         CIGAR errors), per call, SAM order
//   get_read_bases_for_each_target_base + trim_bases_for_homopolymers
//                               alignment.rs:175-201, 364-378 -> k_tile scatter phase (CIGAR walk, right-end trim)
//   Pileup::add_alignment / PileupBase::add_seq   pileup.rs:189-200, 56-65 -> k_tile (counters in shared memory)
//   PileupBase::get_polished_seq + bankers_rounding pileup.rs:67-134, misc.rs:208-215 -> k_tile vote phase
//   polish_one_sequence's join + replace("-","")  polish.rs:185-188 -> k_compact
//
// Design (DESIGN.md §3): the reference's pileup is one counter increment per aligned base into a 80 B/bp array, in read
// order.  Here the alignments are binned by reference position ONCE PER DATASET (k_bin: one 32-byte record + a 256-position bin
// key per alignment; a stable radix sort of (key, alignment index) keeps SAM order inside every bin; k_permute / k_permute_seq
// move records and the bases of the common reads into that order, forward strand), and per polish call ONE persistent kernel
// (k_tile) owns 2048 consecutive positions at a time with every counter of those positions in shared memory, streaming the
// tile's slot range coalesced:
//   * cover[p]   = good alignments whose kept entries include p: interval add (+1 / -1) + in-tile prefix sum;
//   * explicit[p][A,C,G,T], del[p] = entries that differ from the draft base: one shared-memory atomic per mismatch
//     (~0.3 % of bases); count[draft base] = cover - sum(everything explicit); 32-bit counters (pileup.rs:33-37);
//   * alleles other than A,C,G,T,"-" (N / IUPAC bases, insertions): one node per distinct (position, allele) in a
//     per-position chain with an exact count (the reference's HashMap<String,u32>, pileup.rs:40,62);
//   * depth: where every covering alignment has k == 1 the f64 depth equals cover exactly.  Alignments with k != 1 also add
//     2^40 - round(2^40 / k) to a 64-bit fixed-point "deficit" (interval add + prefix sum like cover), so cover - deficit * 2^-40
//     is the depth to within a proven bound (depth_bounds).  The vote only needs depth through four monotone tests; where both
//     ends of the bound give the same answers the vote is the reference's.  Only a 128-position sub-tile with a position whose
//     bound straddles a threshold gets the reference's sequential f64 sum re-done in SAM order, by one warp that merges the
//     (already SAM-ordered) bins overlapping the sub-tile by alignment index (pileup.rs:64, alignment.rs:288);
//   * the vote runs straight out of shared memory: the counters never exist in HBM, nothing has to be zeroed per call but
//     4 B/bp of chain heads, and the working set per CTA does not depend on the assembly size (no L2 cliff).
// Everything is integer / byte work bounded by HBM bandwidth: no tensor cores.
#pragma once

#include "nib_utils.h"
#include "../../include/pp_abi.h"

#define PP_BIN_SHIFT 8               // binning granularity of the alignment sort: 256 reference positions
#define PP_BIN (1u << PP_BIN_SHIFT)
#define PP_SUB_SHIFT 7               // ordered-depth sub-tile: 128 positions (one warp, 4 positions per lane)
#define PP_SUB (1u << PP_SUB_SHIFT)
#define TL_T 2048                    // positions one CTA owns at a time (= the vote / compaction chunk)
#define TL_THREADS 512
#define TL_PER_THREAD (TL_T / TL_THREADS)
#define TL_LONG_E 512                // alignments with more entries than this are not binned: every tile looks at the "long" list
#define TL_QCAP 1024                 // queued reads per tile (more are walked in place)
#define TL_FAST_LEN 192              // longest read the register-resident fast path takes
#define PR_THREADS 256               // k_prep CTA: one alignment per thread
#define SC_GROUP_SCAN_LIMIT 8192     // alignments of one read group a thread will scan outside its block for k
#define VT_THREADS 256
#define VT_ITEMS 8
#define VT_CHUNK (VT_THREADS * VT_ITEMS)
#define NONE32 0xFFFFFFFFu
static_assert(VT_CHUNK == TL_T, "k_tile hands k_compact one chunk per tile");
static_assert(TL_T % PP_BIN == 0 && TL_T / PP_SUB == TL_THREADS / 32 && TL_PER_THREAD * 32 == PP_SUB, "tile = whole bins; warp w owns depth sub-tile w and votes on it");

enum : unsigned {
    ERR_UNKNOWN_CONTIG = 1, ERR_SEQ_MISMATCH = 2, ERR_BAD_OP = 3, ERR_OOB = 4, ERR_NOSEQ = 5,
    ERR_PAST_END = 6                 // (k_bin -> k_past_end only: starts at or past its contig's end; ERR_OOB or nothing once the trim is known)
};
enum : unsigned { FL_NODE_OVF = 1, FL_OUT_OVF = 8, FL_BIGGROUP = 16, FL_PAST_END = 32 };   // FL_PAST_END: k_bin left ERR_PAST_END codes
enum : unsigned { TR_RC = 1, TR_FAST = 2, TR_LONG = 4, TR_FAST1 = 8, TR_STAGED = 16 };   // TR_FAST1: aM bI|bD cM, a in bits 8..15, b in 16..27, D in bit 28
                                                                                      // TR_STAGED: 4-bit, <= 192 bases, not long (bases in sseq)

struct DevStatus {
    unsigned long long err;          // min over (aln << 8 | code); ~0 = none
    unsigned long long n_used;       // good alignments
    unsigned long long out_len;      // polished bases
    unsigned int node_count;         // other-allele nodes allocated
    unsigned int flags;
    unsigned int max_ext;            // (binning) largest entry count of a binned alignment: how many bins a tile looks back
    unsigned int ticket;             // next tile (k_tile's dynamic schedule)
    unsigned int n_changes;          // changed positions k_tile appended to the change list (counted beyond its capacity too)
    unsigned int pad1;
#ifdef PP_TILE_PROF
    unsigned long long prof[12];     // cycles of thread 0 per phase (A, B, queue, C, D+E), queued reads, tiles, largest queue, depth-walk cycles, walks, tiles with a walk,
                                     // cycles lane 0 of every warp waited for its chunks' data in phase B
#endif
};

struct DevParams {                   // pp_polish_params, device resident (refreshed by a memcpy before each call)
    double fv, fi;
    uint32_t min_depth, max_errors;
    int careful;
    int pad;
};

// One distinct other allele at one position (the reference's HashMap<String,u32> entry, pileup.rs:40,62).
struct OthNode {
    unsigned long long sig;          // allele signature (see make_sig)
    unsigned long long val;          // where to read the allele: aln << 32 | start << 16 | len
    uint32_t count;
    uint32_t next;                   // next node of the same position, NONE32 = end
};

// What k_tile needs to know about one alignment that can contribute.  Written once per dataset by k_bin (SAM order) and moved
// into bin order by k_permute; everything in it is independent of the polish options.
struct __align__(16) TileRec {
    uint32_t gstart;                 // global position of the first entry
    uint32_t seq_off;                // PP_SEQ_BLOCK units (queued walks; the chunk loop reads a TR_STAGED slot's own copy of the bases)
    uint32_t cigar_off;
    uint32_t len_nc;                 // seq_len | n_cigar << 16
    uint32_t aln;                    // index in SAM order
    uint32_t E;                      // entries before the trim (saturated)
    uint32_t flags;                  // TR_*
    uint32_t cend;                   // end of the contig (global position)
};
#define TL_SEQ_QUADS 6               // 16-byte quads of a slot's copy of its read (TR_STAGED: <= 192 bases)

struct DevData {                     // everything the kernels read, by value
    // alignments
    unsigned long long n_aln;
    const uint32_t *contig, *ref_start, *read_id, *seq_off, *cigar_off, *nm, *cigar_ops;
    const uint16_t *seq_len, *n_cigar;
    const uint8_t *flags, *seq_pool;
    // assembly
    const uint8_t* draft;            // ASCII
    const unsigned long long* contig_off;
    uint32_t n_contigs;
    uint32_t G;                      // total positions
    uint32_t n_bins;                 // ceil(G / 256); key n_bins = long list, n_bins + 1 = contributes nothing
    uint32_t n_tiles;
    // work
    uint32_t* k;                     // [n_reads] good alignments per read (only in the global-k fallback mode)
    // the dataset in bin order (built once per dataset: k_bin -> stable sort -> k_bin_bounds -> k_permute / k_permute_seq)
    TileRec* recs;                   // [n_aln] SAM order (binning scratch)
    uint32_t *key, *val;             // [n_aln] (bin, alignment) pairs, SAM order (binning scratch)
    const uint32_t* sval;            // [n_aln] alignment indices sorted by bin (stable: SAM order inside a bin)
    uint32_t* bin_start;             // [n_bins + 3] first sorted slot of every bin
    TileRec* srec;                   // [n_slots] records in slot (= bin, then SAM) order
    uint4* sseq;                     // [n_slots * 6] 4-bit mode: every TR_STAGED read again, forward strand, base 0 at nibble 0
    uint32_t n_slots;                // alignments that can contribute (slots before the "nothing" key)
    const uint32_t* tile_order;      // [n_tiles] tiles by decreasing slot count: the ticket order (heavy tiles first, no long tail)
    uint32_t max_ext;                // largest entry count of a binned alignment (how many bins a tile looks back)
    uint8_t* errc;                   // [n_aln] 0, or the error the reference raises IF the alignment is good (alignment.rs:187-198,298-300)
    uint16_t* gq;                    // [n_aln] everything k_goodk needs that does not depend on the options (GQ_* bits; high byte min(NM, 255))
    // per call
    uint32_t* kf;                    // [n_aln] k of the alignment's read group if it contributes under the current options, else 0
    uint4* wrec;                     // [n_aln] per sorted slot: (alignment, first position, kept entries, k) - what the ordered depth walk reads
    uint32_t* oth_head;              // [G] 1 + index of the first OthNode of the position, 0 = none
    OthNode* nodes;
    uint32_t node_cap;
    const DevParams* prm;
    DevStatus* st;
};

// ------------------------------------------------------------------------------------------------------
// small device helpers
// ------------------------------------------------------------------------------------------------------
__device__ __forceinline__ void report_error(DevStatus* st, unsigned long long aln, unsigned code) {
    atomicMin(&st->err, (aln << 8) | (unsigned long long)code);
}

#if defined(PP_EMULATE)
static uint8_t c_comp[256];
static const char c_nib2asc[16] = {'=', 'A', 'C', 'M', 'G', 'R', 'S', 'V', 'T', 'W', 'Y', 'H', 'K', 'D', 'B', 'N'};
#else
__constant__ uint8_t c_comp[256];      // misc.rs:170-182 complement_base on upper-cased bytes
__constant__ char c_nib2asc[16] = {'=', 'A', 'C', 'M', 'G', 'R', 'S', 'V', 'T', 'W', 'Y', 'H', 'K', 'D', 'B', 'N'};
#endif

#if defined(PP_EMULATE)
// Directed rounding on the CPU: the round-to-nearest result, stepped one ulp in the rounding direction when the exact result
// (its error term from TwoSum / FMA) lies beyond it.
static inline double emu_step(double r, double err, bool up) {
    return (up ? err > 0.0 : err < 0.0) ? std::nextafter(r, up ? INFINITY : -INFINITY) : r;
}
static inline double emu_add(double a, double b, bool up) {
    volatile double r = a + b;
    const double bv = r - a, err = (a - (r - bv)) + (b - bv);
    return emu_step(r, err, up);
}
static inline double __dadd_ru(double a, double b) { return emu_add(a, b, true); }
static inline double __dsub_rd(double a, double b) { return emu_add(a, -b, false); }
static inline double __dsub_ru(double a, double b) { return emu_add(a, -b, true); }
static inline double __dmul_ru(double a, double b) { volatile double r = a * b; return emu_step(r, std::fma(a, b, -r), true); }
static inline double emu_ull2double(unsigned long long x, bool up) {
    const double r = (double)x;                               // round to nearest
    const bool above = r >= 18446744073709551616.0 || (unsigned long long)r > x, below = r < 18446744073709551616.0 && (unsigned long long)r < x;
    if (up ? below : above) return std::nextafter(r, up ? INFINITY : -INFINITY);
    return r;
}
static inline double __ull2double_rd(unsigned long long x) { return emu_ull2double(x, false); }
static inline double __ull2double_ru(unsigned long long x) { return emu_ull2double(x, true); }
static inline double __ull2double_rn(unsigned long long x) { return (double)x; }
// Reads the chunk loop handed to the general walk from the pool (queued, or walked in place when the queue is full), summed over
// the tiles that look at them: the emulator's tests read the exported symbol to see how many reads the staged walk left behind.
inline std::atomic<unsigned long long> emu_n_queued{0};
#endif

__device__ __forceinline__ uint32_t brev4(uint32_t c) {   // complement of a BAM nibble = 4-bit reversal
    return __brev(c) >> 28;
}

// mask of the n lowest nibbles of a 64-bit word, n clamped to [0, 16]
__device__ __forceinline__ unsigned long long nibmask(int n) {
    return n <= 0 ? 0ull : (n >= 16 ? ~0ull : ((1ull << (4 * n)) - 1ull));
}

// Sequence access policies.  sym = 4-bit code (SEQ4) or upper-cased ASCII byte (SEQ8).
template <int BITS> struct Seq;
template <> struct Seq<4> {
    static __device__ __forceinline__ uint32_t read_sym(const uint8_t* pool, uint32_t off_blk, uint32_t len, bool rc, uint32_t i) {
        uint32_t j = rc ? (len - 1 - i) : i;
        uint32_t b = pool[(size_t)off_blk * (PP_SEQ_BLOCK / 2) + (j >> 1)];
        uint32_t c = (b >> ((j & 1) * 4)) & 15u;
        return rc ? brev4(c) : c;
    }
    static __device__ __forceinline__ bool is_del(uint32_t) { return false; }
    static __device__ __forceinline__ int acgt(uint32_t s) { return s == 1 ? 0 : s == 2 ? 1 : s == 4 ? 2 : s == 8 ? 3 : -1; }
    static __device__ __forceinline__ uint8_t ascii(uint32_t s) { return (uint8_t)c_nib2asc[s & 15]; }
};
template <> struct Seq<8> {
    static __device__ __forceinline__ uint32_t read_sym(const uint8_t* pool, uint32_t off_blk, uint32_t len, bool rc, uint32_t i) {
        uint32_t j = rc ? (len - 1 - i) : i;
        uint32_t b = pool[(size_t)off_blk * PP_SEQ_BLOCK + j];
        return rc ? c_comp[b] : b;
    }
    static __device__ __forceinline__ bool is_del(uint32_t s) { return s == '-'; }   // the 1-char string "-"
    static __device__ __forceinline__ int acgt(uint32_t s) { return s == 'A' ? 0 : s == 'C' ? 1 : s == 'G' ? 2 : s == 'T' ? 3 : -1; }
    static __device__ __forceinline__ uint8_t ascii(uint32_t s) { return (uint8_t)s; }
};

// Allele signature of an "other" allele (anything that is not a single A/C/G/T or "-"): the whole string for
// short alleles (4-bit: <= 15 bases, 8-bit: <= 7 bytes) with the length in the low field, else length field 0
// and a hash of the content (equality then falls back to comparing the sequences themselves).
template <int BITS> __device__ __forceinline__ bool sig_exact(unsigned long long sig) {
    return BITS == 4 ? (sig & 15ull) != 0 : (sig & 255ull) != 0;
}
// (bs: where the read's bases are, PoolBases / StagedBases)
template <int BITS, class Bases>
__device__ __forceinline__ unsigned long long make_sig(const Bases& bs, uint32_t start, uint32_t len) {
    const uint32_t maxlen = BITS == 4 ? 15 : 7;
    if (len <= maxlen) {
        unsigned long long sig = len;
        for (uint32_t i = 0; i < len; ++i)
            sig |= (unsigned long long)bs.sym(start + i) << ((BITS == 4 ? 4 : 8) * (i + 1));
        return sig;
    }
    unsigned long long h = 0xcbf29ce484222325ull;
    for (uint32_t i = 0; i < len; ++i) { h ^= bs.sym(start + i); h *= 0x100000001b3ull; }
    h ^= len;
    return h << (BITS == 4 ? 4 : 8);
}

__device__ __forceinline__ uint32_t asc2nib(uint32_t c) {   // ASCII draft base -> BAM code, 0 = not one of the 15 letters (never equals a read code)
    // codes of 'A'..'P' (lo) and 'Q'..'Z' (hi), four bits per letter: A1 B14 C2 D13 G4 H11 K12 M3 N15 | R5 S6 T8 V7 W9 Y10
    const unsigned long long lo = 0xf30c00b400d2e1ull, hi = 0xa09708650ull;
    const uint32_t i = c - 'A';
    return i < 26u ? (uint32_t)((i < 16u ? lo >> (4 * i) : hi >> (4 * (i - 16u))) & 15ull) : 0u;
}

// block-wide exclusive scan of one u64 per thread (NT threads); returns exclusive prefix, total in *total
template <int NT>
__device__ __forceinline__ unsigned long long block_exscan(unsigned long long v, unsigned long long* s_warp, unsigned long long* total) {
    const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    unsigned long long inc = v;
    for (int o = 1; o < 32; o <<= 1) {
        unsigned long long t = __shfl_up_sync(0xffffffffu, inc, o);
        if ((int)lane >= o) inc += t;
    }
    if (lane == 31) s_warp[warp] = inc;
    __syncthreads();
    if (warp == 0) {
        unsigned long long w = (lane < NT / 32) ? s_warp[lane] : 0;
        unsigned long long winc = w;
        for (int o = 1; o < 32; o <<= 1) {
            unsigned long long t = __shfl_up_sync(0xffffffffu, winc, o);
            if ((int)lane >= o) winc += t;
        }
        if (lane < NT / 32) s_warp[lane] = winc - w;      // exclusive per-warp offsets
        if (lane == 31) *total = winc;
    }
    __syncthreads();
    unsigned long long r = s_warp[warp] + inc - v;
    __syncthreads();
    return r;
}

// misc.rs:208-215 bankers_rounding on a non-negative finite double (depth * fraction)
__device__ __forceinline__ uint32_t bankers_rounding(double x) {
    uint32_t rd;
    if (!(x == x) || x <= 0.0) rd = 0;
    else if (x >= 4294967295.0) rd = 4294967295u;
    else rd = (uint32_t)x;                                  // truncation
    const double fr = __dsub_rn(x, trunc(x));
    if (fr < 0.5) return rd;
    if (fr > 0.5) return rd + 1;
    return rd + (rd & 1u);
}

// Everything the vote reads from depth (pileup.rs:70-72, 76): the valid and invalid thresholds and the low-depth test.  All three
// are monotone non-decreasing in depth (IEEE multiplication by a non-negative constant and bankers_rounding both are).
struct Thresholds { uint32_t vt, it; bool low; };
__device__ __forceinline__ Thresholds vote_thresholds(const DevParams& prm, double depth) {
    return Thresholds{max(prm.min_depth, bankers_rounding(__dmul_rn(depth, prm.fv))), bankers_rounding(__dmul_rn(depth, prm.fi)),
                      depth < (double)prm.min_depth};
}
__device__ __forceinline__ bool same_thresholds(const DevParams& prm, double a, double b) {
    const Thresholds x = vote_thresholds(prm, a), y = vote_thresholds(prm, b);
    return x.vt == y.vt && x.it == y.it && x.low == y.low;
}

// The depth of a position from its cover (n covering alignments, an exact integer) and its fixed-point deficit M = sum over the
// covering alignments with k != 1 of 2^40 - r_k, r_k = round(2^40 / k) (depth_deficit).  The reference's depth d_ref is the
// sequential f64 sum, in SAM order, of fl(1/k) over the covering alignments; T = sum of 1/k is the exact value.
//   * fixed point: |r_k 2^-40 - 1/k| <= 2^-41 and the k == 1 terms are exact, so d_fx = n - M 2^-40 has |d_fx - T| <= m 2^-41,
//     m = covering alignments with k != 1 <= n;
//   * the reference: fl(1/k) = (1/k)(1 + e), |e| <= u = 2^-53, then n - 1 additions of non-negative terms, so
//     |d_ref - T| <= gamma_n T with gamma_n = n u / (1 - n u) (Higham, Accuracy and Stability, Lemma 3.1 and §4.2), and T <= n;
//     for n u <= 1/2, gamma_n T <= 2 n^2 u = n^2 2^-52;
//   * so |d_ref - d_fx| <= E = n 2^-41 + n^2 2^-52, and d_fx itself is bracketed by converting M to double rounded down and up
//     (scaling by 2^-40 is exact).  Every step below rounds outwards, so [lo, hi] contains d_ref.
// M < 2^63 (no wrap of the 64-bit prefix sum) needs m < 2^23: positions with n >= TL_DEF_COVER are not bounded here.
#define TL_DEF_COVER (1u << 23)
struct DepthBounds { double lo, hi, fx; };
__device__ __forceinline__ DepthBounds depth_bounds(uint32_t cover, unsigned long long deficit) {
    const double n = (double)cover;
    const double e = __dadd_ru(n * 0x1p-41, __dmul_ru(n, n) * 0x1p-52);
    DepthBounds b;
    b.lo = __dsub_rd(__dsub_rd(n, __ull2double_ru(deficit) * 0x1p-40), e);
    b.hi = __dadd_ru(__dsub_ru(n, __ull2double_rd(deficit) * 0x1p-40), e);
    b.fx = __dsub_rn(n, __ull2double_rn(deficit) * 0x1p-40);
    return b;
}
__device__ __forceinline__ unsigned long long depth_deficit(uint32_t k) {   // 2^40 - round(2^40 / k), k >= 2
    return (1ull << 40) - ((1ull << 40) + k / 2) / k;
}

// ------------------------------------------------------------------------------------------------------
// Goodness (alignment.rs:283-287) and --careful (:277-279) of one alignment.  `multi` = its read group has more
// than one aligned record.
// ------------------------------------------------------------------------------------------------------
__device__ __forceinline__ bool group_is_multi(const DevData& d, unsigned long long a, uint32_t rid) {
    return (a > 0 && d.read_id[a - 1] == rid) || (a + 1 < d.n_aln && d.read_id[a + 1] == rid);
}
__device__ __forceinline__ bool alignment_is_good(const DevData& d, unsigned long long a, bool multi, uint32_t co, uint32_t nc, uint8_t fl) {
    if (nc == 0) { report_error(d.st, a, ERR_BAD_OP); return false; }       // the packer never emits this
    const uint32_t f = d.cigar_ops[co] & 15u, l = d.cigar_ops[co + nc - 1] & 15u;
    return (f == PP_OP_M || f == PP_OP_EQ) && (l == PP_OP_M || l == PP_OP_EQ) && d.nm[a] <= d.prm->max_errors &&
           !(fl & PP_FLAG_ZPFAIL) && !(d.prm->careful && multi);
}

// The same from the per-alignment summary k_bin leaves behind (written once per dataset): bit 0 first and last CIGAR op are M / =,
// 1 ZP:Z:fail, 2 ghost, 3 the read group has more than one aligned record, 4 no CIGAR ops at all, 5..7 the error a GOOD alignment
// raises (errc), 8..15 min(NM, 255).
#define GQ_ENDS 1u
#define GQ_ZP 2u
#define GQ_GHOST 4u
#define GQ_MULTI 8u
#define GQ_NOOPS 16u
__device__ __forceinline__ bool good_from_summary(const DevData& d, const DevParams& prm, unsigned long long a, uint32_t q) {
    if (q & GQ_NOOPS) { report_error(d.st, a, ERR_BAD_OP); return false; }             // the packer never emits this
    uint32_t nm = q >> 8;
    if (nm == 255u && prm.max_errors >= 255u) nm = d.nm[a];
    return (q & GQ_ENDS) && nm <= prm.max_errors && !(q & GQ_ZP) && !(prm.careful && (q & GQ_MULTI));
}

// k_classify_multi: FALLBACK pre-pass, only launched when a read group was too large for k_prep's in-kernel scan
// (FL_BIGGROUP): k = #good of every multi-record group into a global array (alignment.rs:288).
__global__ void __launch_bounds__(256) k_classify_multi(DevData d) {
    for (unsigned long long a = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x; a < d.n_aln;
         a += (unsigned long long)gridDim.x * blockDim.x) {
        const uint32_t rid = d.read_id[a];
        if (!group_is_multi(d, a, rid)) continue;
        if (alignment_is_good(d, a, true, d.cigar_off[a], d.n_cigar[a], d.flags[a])) atomicAdd(&d.k[rid], 1u);
    }
}

// ------------------------------------------------------------------------------------------------------
// Once per dataset: k_bin.  One alignment per thread, every input array read coalesced: the 256-position bin of its first
// entry (or "long" / "can never contribute") and the record k_tile will read, none of which depends on the polish options.
// ------------------------------------------------------------------------------------------------------
template <int BITS>
__device__ __forceinline__ void bin_body(const DevData& d) {
    uint32_t max_ext = 0;
    bool pending = false;                                       // an alignment of this thread starts at or past its contig's end
    for (unsigned long long aln = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x; aln < d.n_aln; aln += (unsigned long long)gridDim.x * blockDim.x) {
        uint32_t key = d.n_bins + 1;                            // can never contribute (k_goodk raises `err` if it is "good")
        uint32_t err = 0;
        const uint32_t c = d.contig[aln];
        const uint8_t fl = d.flags[aln];
        const uint32_t ncig = d.n_cigar[aln], cigoff = d.cigar_off[aln];
        if (c == PP_CONTIG_UNKNOWN) err = ERR_UNKNOWN_CONTIG;                      // alignment.rs:298-300
        else if (fl & PP_FLAG_NOSEQ) err = ERR_NOSEQ;
        else if (ncig == 0) err = ERR_BAD_OP;                                      // the packer never emits this
        else {
            const unsigned long long gs = d.contig_off[c] + d.ref_start[aln];
            const unsigned long long ce = d.contig_off[c + 1];
            const uint32_t len = d.seq_len[aln];
            // E = entries (one per consumed reference position), R = read bases consumed (alignment.rs:175-198)
            unsigned long long E = 0, R = 0;
            bool bad = false;
            const uint32_t* ops = d.cigar_ops + cigoff;
            for (uint32_t p = 0; p < ncig; ++p) {
                const uint32_t op = ops[p], o = op & 15u, l = op >> 4;
                if (o == PP_OP_M || o == PP_OP_EQ || o == PP_OP_X) { E += l; R += l; }
                else if (o == PP_OP_I) R += l;
                else if (o == PP_OP_D) E += l;
                else bad = true;                                                   // alignment.rs:187-193
            }
            // the reference checks the ops, then the length, and only then indexes the pileup - for the entries the trim keeps
            if (bad) err = ERR_BAD_OP;
            else if (R != len) err = ERR_SEQ_MISMATCH;                             // :195-198
            else if (gs >= ce) {
                // starts at or past the end: an overrun unless the trim removes every entry (pileup.rs:189-200).  The bases may still be
                // on their way to the device, so k_past_end decides once they are there.
                if (!(fl & PP_FLAG_GHOST)) { err = ERR_PAST_END; pending = true; }
            } else if (!(fl & PP_FLAG_GHOST) && len != 0) {
                const bool is_long = E > TL_LONG_E;
                const uint32_t f0 = ops[0] & 15u;
                const bool fast = BITS == 4 && ncig == 1 && (f0 == PP_OP_M || f0 == PP_OP_EQ) && len <= TL_FAST_LEN;
                // every other short 4-bit read is walked by the general walk from its staged bases, in the chunk loop
                const bool staged = BITS == 4 && len <= TL_FAST_LEN && !is_long;
                uint32_t flags = ((fl & PP_FLAG_RC) ? TR_RC : 0u) | (fast ? TR_FAST : 0u) | (is_long ? TR_LONG : 0u) | (staged ? TR_STAGED : 0u);
                if (BITS == 4 && ncig == 3 && len <= TL_FAST_LEN && !is_long) {
                    // one insertion or one deletion between two match runs: aM bI cM / aM bD cM (the fast walk hands the read to the
                    // general walk when its trim reaches past the last run)
                    const uint32_t o1 = ops[1] & 15u, o2 = ops[2] & 15u, la = ops[0] >> 4, lb2 = ops[1] >> 4, lc = ops[2] >> 4;
                    if ((f0 == PP_OP_M || f0 == PP_OP_EQ) && (o1 == PP_OP_I || o1 == PP_OP_D) && (o2 == PP_OP_M || o2 == PP_OP_EQ) &&
                        la >= 1 && la <= 255 && lb2 >= 1 && lb2 <= 4095 && lc >= 1)
                        flags |= TR_FAST | TR_FAST1 | (la << 8) | (lb2 << 16) | (o1 == PP_OP_D ? 1u << 28 : 0u);
                }
                uint4* dst = reinterpret_cast<uint4*>(d.recs + aln);
                dst[0] = make_uint4((uint32_t)gs, d.seq_off[aln], cigoff, len | (ncig << 16));
                dst[1] = make_uint4((uint32_t)aln, (uint32_t)min(E, 0xFFFFFFFFull), flags, (uint32_t)ce);
                key = is_long ? d.n_bins : (uint32_t)(gs >> PP_BIN_SHIFT);
                if (!is_long) max_ext = max(max_ext, (uint32_t)E);
            }
        }
        d.errc[aln] = (uint8_t)err;
        {
            uint32_t q = (fl & PP_FLAG_ZPFAIL ? GQ_ZP : 0u) | (fl & PP_FLAG_GHOST ? GQ_GHOST : 0u) | (ncig == 0 ? GQ_NOOPS : 0u) | (err << 5) |
                         (min(d.nm[aln], 255u) << 8);
            if (ncig) {
                const uint32_t f = d.cigar_ops[cigoff] & 15u, l = d.cigar_ops[cigoff + ncig - 1] & 15u;
                if ((f == PP_OP_M || f == PP_OP_EQ) && (l == PP_OP_M || l == PP_OP_EQ)) q |= GQ_ENDS;
            }
            if (group_is_multi(d, aln, d.read_id[aln])) q |= GQ_MULTI;
            d.gq[aln] = (uint16_t)q;
        }
        d.key[aln] = key; d.val[aln] = (uint32_t)aln;
    }
    for (int o = 16; o > 0; o >>= 1) max_ext = max(max_ext, __shfl_down_sync(0xffffffffu, max_ext, o));
    if ((threadIdx.x & 31) == 0 && max_ext) atomicMax(&d.st->max_ext, max_ext);
    if (pending) atomicOr(&d.st->flags, (unsigned)FL_PAST_END);
}

// Slot i of the binned dataset: the record of the alignment the stable sort put there.
__device__ __forceinline__ void permute_body(const DevData& d) {
    const unsigned long long i = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= d.n_slots) return;
    const uint4* src = reinterpret_cast<const uint4*>(d.recs + d.sval[i]);
    uint4* dst = reinterpret_cast<uint4*>(d.srec + i);
    dst[0] = src[0]; dst[1] = src[1];
}

// ... and its bases (4-bit mode, TR_STAGED reads): the EFFECTIVE read - the stored one, or its reverse complement for
// PP_FLAG_RC records (alignment.rs:161-167: complementing a BAM nibble = reversing its 4 bits, so the whole thing is one bit
// reversal) - forward, base 0 at nibble 0, zero padded to 192 bases.  One thread per 16-byte quad (32 bases).
__device__ __forceinline__ void permute_seq_body(const DevData& d) {
    const unsigned long long t = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x;
    const unsigned long long i = t / TL_SEQ_QUADS;
    const uint32_t g = (uint32_t)(t % TL_SEQ_QUADS);
    if (i >= d.n_slots) return;
    const TileRec& r = d.srec[i];
    if (!(r.flags & TR_STAGED)) return;                         // the queued general walk reads the pool itself
    const uint32_t len = r.len_nc & 0xFFFFu, nw = (len + 7) >> 3;                         // words that hold bases
    const uint32_t* s32 = reinterpret_cast<const uint32_t*>(d.seq_pool + (size_t)r.seq_off * 16);
    uint32_t out[4];
    if (!(r.flags & TR_RC)) {
        const uint4 q = *reinterpret_cast<const uint4*>(s32 + 4 * g);                       // (reads past the last word stay inside the padded pool)
        out[0] = q.x; out[1] = q.y; out[2] = q.z; out[3] = q.w;
    } else {
        // effective nibble e = complement of stored nibble len-1-e = nibble (8 nw - len + e) of the word-reversed, bit-reversed words
        const uint32_t pad = 8 * nw - len;                      // 0 .. 7
        uint32_t v[5];
#pragma unroll
        for (int w = 0; w < 5; ++w) { const uint32_t x = 4 * g + (uint32_t)w; v[w] = x < nw ? __brev(s32[nw - 1 - x]) : 0u; }
#pragma unroll
        for (int w = 0; w < 4; ++w) out[w] = __funnelshift_r(v[w], v[w + 1], pad * 4);
    }
#pragma unroll
    for (int w = 0; w < 4; ++w) {
        const uint32_t m = 4 * g + (uint32_t)w;
        if (m >= nw) out[w] = 0;
        else if (m == nw - 1 && (len & 7)) out[w] &= 0xFFFFFFFFu >> ((8 - (len & 7)) * 4);  // nothing but zeros past the last base
    }
    d.sseq[t] = make_uint4(out[0], out[1], out[2], out[3]);
}

// Slots a tile has to look at (its own bins + the look-back): the weight the tiles are handed out by, heaviest first.
__device__ __forceinline__ void tile_weight_body(const DevData& d, uint32_t* __restrict__ weight, uint32_t* __restrict__ index) {
    const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= d.n_tiles) return;
    const uint32_t lb = (d.max_ext + PP_BIN - 1) >> PP_BIN_SHIFT;
    const uint32_t b0 = (t * (uint32_t)TL_T) >> PP_BIN_SHIFT;
    weight[t] = d.bin_start[min(b0 + (uint32_t)(TL_T / PP_BIN), d.n_bins)] - d.bin_start[b0 >= lb ? b0 - lb : 0u];
    index[t] = t;
}
#if !defined(PP_EMULATE)
__global__ void __launch_bounds__(256) k_tile_weight(DevData d, uint32_t* __restrict__ weight, uint32_t* __restrict__ index) { tile_weight_body(d, weight, index); }
#endif

// ------------------------------------------------------------------------------------------------------
// Per call: k_goodk = process_one_read (alignment.rs:275-305) for every alignment, one per thread, SAM order, coalesced:
// goodness under the current options, k = good records of the consecutive-QNAME group, --careful, and the errors the reference
// raises for a good alignment.  kf[aln] = k if the alignment adds to the pileup, else 0.
// GLOBALK = false: k of a multi-record group is counted right here (its records are consecutive alignments);
// GLOBALK = true: k comes from k_classify_multi (fallback for huge groups).
// ------------------------------------------------------------------------------------------------------
// (four alignments per thread with 16-byte loads were measured slower than this one-per-thread form)
struct PrepShared {
    uint32_t rid[PR_THREADS];
    uint8_t good[PR_THREADS];
    uint32_t n_good;
};

template <bool GLOBALK>
__device__ __forceinline__ void goodk_body(const DevData& d, PrepShared& sh) {
    const uint32_t tid = threadIdx.x, lane = tid & 31;
    const unsigned long long n_blocks = (d.n_aln + PR_THREADS - 1) / PR_THREADS;
    const DevParams prm = *d.prm;
    unsigned long long used = 0;
    for (unsigned long long blk = blockIdx.x; blk < n_blocks; blk += gridDim.x) {
        const unsigned long long blk0 = blk * PR_THREADS;
        const unsigned long long aln = blk0 + tid;
        const uint32_t nvalid = (uint32_t)min((unsigned long long)PR_THREADS, d.n_aln - blk0);
        bool good = false, grp = false;
        uint32_t rid = 0, q = 0;
        if (aln < d.n_aln) {
            rid = d.read_id[aln];
            q = d.gq[aln];                                      // 6 bytes per alignment in all: the rest was settled by k_bin
            grp = q & GQ_MULTI;
            good = good_from_summary(d, prm, aln, q);
        }
        sh.rid[tid] = rid;
        sh.good[tid] = good ? 1 : 0;
        __syncthreads();
        // k = number of good alignments of the read group (alignment.rs:288)
        uint32_t k = 1;
        if (good && grp) {
            if (GLOBALK) k = d.k[rid];
            else {
                uint32_t count = 1, steps = 0;
                int i = (int)tid;
                while (i > 0 && sh.rid[i - 1] == rid) { --i; count += sh.good[i]; }
                if (i == 0) {
                    for (unsigned long long a2 = blk0; a2 > 0 && d.read_id[a2 - 1] == rid;) {
                        --a2;
                        count += good_from_summary(d, prm, a2, d.gq[a2]) ? 1 : 0;
                        if (++steps > SC_GROUP_SCAN_LIMIT) { atomicOr(&d.st->flags, (unsigned)FL_BIGGROUP); break; }
                    }
                }
                i = (int)tid;
                while (i + 1 < (int)nvalid && sh.rid[i + 1] == rid) { ++i; count += sh.good[i]; }
                if (i == (int)nvalid - 1) {
                    for (unsigned long long a2 = blk0 + nvalid - 1; a2 + 1 < d.n_aln && d.read_id[a2 + 1] == rid;) {
                        ++a2;
                        count += good_from_summary(d, prm, a2, d.gq[a2]) ? 1 : 0;
                        if (++steps > SC_GROUP_SCAN_LIMIT) { atomicOr(&d.st->flags, (unsigned)FL_BIGGROUP); break; }
                    }
                }
                k = count;
            }
        }
        if (q & GQ_GHOST) good = false;                         // another shard scatters it; it only counted towards k
        uint32_t kf = 0;
        if (good) {
            used++;
            const uint32_t e = (q >> 5) & 7u;                   // what the reference raises for a good alignment (found once, by k_bin)
            if (e) report_error(d.st, aln, e);
            else kf = k;
        }
        if (aln < d.n_aln) d.kf[aln] = kf;
        __syncthreads();
    }
    // good alignments (alignment.rs:304): block reduce, one atomic per CTA
    if (tid == 0) sh.n_good = 0;
    __syncthreads();
    for (int o = 16; o > 0; o >>= 1) used += __shfl_down_sync(0xffffffffu, used, o);
    if (lane == 0 && used) atomicAdd(&sh.n_good, (uint32_t)used);
    __syncthreads();
    if (tid == 0 && sh.n_good) atomicAdd(&d.st->n_used, (unsigned long long)sh.n_good);
}

#if !defined(PP_EMULATE)
template <int BITS> __global__ void __launch_bounds__(256) k_bin(DevData d) { bin_body<BITS>(d); }
__global__ void __launch_bounds__(256) k_permute(DevData d) { permute_body(d); }
__global__ void __launch_bounds__(256) k_permute_seq(DevData d) { permute_seq_body(d); }
template <bool GLOBALK>
__global__ void __launch_bounds__(PR_THREADS) k_goodk(DevData d) {
    __shared__ PrepShared sh;
    goodk_body<GLOBALK>(d, sh);
}
#endif

// bin_start[b] = first sorted slot whose key is >= b, for b in [0, n_bins + 2] (keys sorted ascending, n of them)
__device__ __forceinline__ void bin_bounds_body(const uint32_t* __restrict__ skey, uint32_t n, uint32_t n_keys, uint32_t* __restrict__ bin_start) {
    const unsigned long long i = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i > n) return;
    const uint32_t hi = (i == n) ? n_keys : min(skey[i], n_keys);          // bins (lo, hi] start at slot i
    const uint32_t lo1 = (i == 0) ? 0u : min(skey[i - 1] + 1u, n_keys + 1u);
    for (uint32_t b = lo1; b <= hi; ++b) bin_start[b] = (uint32_t)i;
}
#if !defined(PP_EMULATE)
__global__ void __launch_bounds__(256) k_bin_bounds(const uint32_t* __restrict__ skey, uint32_t n, uint32_t n_keys, uint32_t* __restrict__ bin_start) {
    bin_bounds_body(skey, n, n_keys, bin_start);
}
#endif

// ------------------------------------------------------------------------------------------------------
// Other alleles: find-or-insert into the per-position chain.  Nodes are written completely, fenced, then linked
// with a CAS on the head; readers load head and node fields through L2 (ld.cg), so a linked node is always whole.
// ------------------------------------------------------------------------------------------------------
struct SeqRef {                      // where an alignment's bases live, for comparing long alleles
    const uint8_t* seq_pool;
    const uint32_t* seq_off;
    const uint16_t* seq_len;
    const uint8_t* flags;
};

template <int BITS>
__device__ __forceinline__ uint32_t allele_sym(const SeqRef& r, unsigned long long val, uint32_t t) {
    const uint32_t aln = (uint32_t)(val >> 32), start = (uint32_t)(val >> 16) & 0xFFFFu;
    return Seq<BITS>::read_sym(r.seq_pool, r.seq_off[aln], r.seq_len[aln], r.flags[aln] & PP_FLAG_RC, start + t);
}
template <int BITS>
__device__ bool allele_equal(const SeqRef& r, unsigned long long va, unsigned long long vb) {
    const uint32_t la = (uint32_t)va & 0xFFFFu, lb = (uint32_t)vb & 0xFFFFu;
    if (la != lb) return false;
    for (uint32_t i = 0; i < la; ++i)
        if (allele_sym<BITS>(r, va, i) != allele_sym<BITS>(r, vb, i)) return false;
    return true;
}

template <int BITS>
__device__ void other_insert(const DevData& d, uint32_t pos, unsigned long long val, unsigned long long sig) {
    const SeqRef sr{d.seq_pool, d.seq_off, d.seq_len, d.flags};
    uint32_t mine = NONE32;
    uint32_t h = __ldcg(&d.oth_head[pos]);                      // 1 + node index, 0 = empty
    uint32_t stop = 0;
    for (;;) {
        for (uint32_t n = h; n != stop;) {
            const OthNode* nd = &d.nodes[n - 1];
            const unsigned long long nsig = __ldcg(&nd->sig);
            if (nsig == sig && (sig_exact<BITS>(sig) || allele_equal<BITS>(sr, __ldcg(&nd->val), val))) {
                atomicAdd(&d.nodes[n - 1].count, 1u);
                return;                                         // (a node allocated on an earlier round stays unlinked)
            }
            const uint32_t nx = __ldcg(&nd->next);
            n = (nx == NONE32) ? 0 : nx + 1;
        }
        if (mine == NONE32) {
            mine = atomicAdd(&d.st->node_count, 1u);
            if (mine >= d.node_cap) { atomicOr(&d.st->flags, (unsigned)FL_NODE_OVF); return; }
            d.nodes[mine].sig = sig;
            d.nodes[mine].val = val;
            d.nodes[mine].count = 1;
        }
        d.nodes[mine].next = (h == 0) ? NONE32 : h - 1;
        __threadfence();
        const uint32_t old = atomicCAS(&d.oth_head[pos], h, mine + 1);
        if (old == h) return;
        stop = h;                                               // someone linked new nodes in front: look only at those
        h = old;
    }
}

// ------------------------------------------------------------------------------------------------------
// The vote (pileup.rs:67-134)
// ------------------------------------------------------------------------------------------------------
struct VoteParams {
    uint32_t n_chunks;
    uint8_t* out;
    unsigned long long out_cap;
    unsigned long long* out_off;     // [n_contigs+1]
    unsigned long long *changed, *zero_depth;   // [n_contigs]
    double* total_depth;             // [n_contigs] sum of the per-position depths (polish.rs:177; the log's mean read depth)
    // per-position verdicts handed from k_tile to k_compact
    uint16_t* res;                    // [padG] low byte = character, high byte = output length (255: see rec_at)
    uint32_t* rec_at;                 // [G] other-allele node to emit at a position (only where res says so)
    long long* chunk_delta;           // [n_chunks] sum(output length) - positions of the chunk
    pp_debug_pos* dbg;                // [G] per-position debug records, or nullptr
    // --changes: the record of every position whose status is changed, appended in no particular order, or nullptr.  Only such
    // positions can emit another base than the draft's, and every one of them reaches the vote (the shortcuts skip only positions
    // that keep their base), so the list costs one atomic per changed position.
    pp_debug_pos* chg;                // [chg_cap]
    uint32_t* chg_pos;                // [chg_cap] global position of each record
    unsigned int* chg_n;              // records appended (DevStatus::n_changes); more than chg_cap: the list overflowed
    uint32_t chg_cap;
};

// What the other-allele slow path needs, passed by value so that the kernel parameter structs are never
// spilled to local memory for a call.
struct OthCtx {
    const OthNode* nodes;
    const uint32_t* head;
    SeqRef sr;
};

struct Tally { uint32_t nvalid, ninter; int which; uint32_t rec; };   // which: 0..3 ACGT, 4 "-", 5 draft's own non-ACGT base, 6 other node

__device__ __forceinline__ void tally(Tally& t, uint32_t c, uint32_t vt, uint32_t it, int which, uint32_t rec) {
    if (c >= vt) { t.nvalid++; t.which = which; t.rec = rec; }
    else if (c >= it) t.ninter++;
}

// Other alleles at `pos` (pileup.rs:102-109): one chain node per distinct allele, count already exact.
__device__ __noinline__ Tally tally_others(OthCtx oc, uint32_t pos, uint32_t vt, uint32_t it, Tally t) {
    for (uint32_t n = oc.head[pos]; n != 0;) {
        const OthNode& nd = oc.nodes[n - 1];
        tally(t, nd.count, vt, it, 6, n - 1);
        n = (nd.next == NONE32) ? 0 : nd.next + 1;
    }
    return t;
}

// Character t of other-allele node `rec` (from the exact signature when there is one, else from the read).
template <int BITS>
__device__ __forceinline__ uint8_t other_char(const OthCtx& oc, uint32_t rec, uint32_t t) {
    const unsigned long long sig = oc.nodes[rec].sig;
    if (sig_exact<BITS>(sig)) return Seq<BITS>::ascii((uint32_t)(sig >> ((BITS == 4 ? 4 : 8) * (t + 1))) & (BITS == 4 ? 15u : 255u));
    return Seq<BITS>::ascii(allele_sym<BITS>(oc.sr, oc.nodes[rec].val, t));
}

// Result of one position, packed: bits 0..15 output length, 16..23 output char (when length is 1 and not from a
// multi-base node), bit 24 changed, bit 25 emit from node `rec`.
struct PosOut { uint32_t packed; uint32_t rec; };

// The debug record of one voted position (what get_debug_line prints, pileup.rs:137-166).
__device__ __forceinline__ void debug_record(pp_debug_pos* r, double depth, uint32_t vt, uint32_t it, uint32_t cA, uint32_t cC, uint32_t cG,
                                             uint32_t cT, uint32_t cDel, uint32_t matched, uint32_t n_other, uint32_t orig, uint32_t status, PosOut o) {
    r->depth = depth; r->valid_threshold = vt; r->invalid_threshold = it;
    r->count[0] = cA; r->count[1] = cC; r->count[2] = cG; r->count[3] = cT; r->count[4] = cDel; r->count[5] = matched;
    r->n_other = n_other;
    r->new_node = ((o.packed >> 25) & 1u) ? o.rec : 0xFFFFFFFFu;
    r->original = (uint8_t)orig; r->status = (uint8_t)status;
    r->new_char = ((o.packed >> 25) & 1u) ? 0 : (((o.packed & 0xFFFFu) == 0 && orig != '-') ? (uint8_t)'-' : (uint8_t)(o.packed >> 16));
}

// The vote of pileup.rs:67-134 for one covered position.  packed bits 26..28 carry the BaseStatus.  `depth` must be the
// reference's own where a record is written (vp.dbg, or CHG and the position changes): the records print it.
template <int BITS, bool CHG>
__device__ __forceinline__ PosOut vote_position(const OthCtx& oc, const DevParams& prm, uint32_t pos, uint32_t orig, double depth,
                                                uint32_t cA, uint32_t cC, uint32_t cG, uint32_t cT, uint32_t cDel,
                                                uint32_t matched, uint32_t n_other, const VoteParams& vp) {
    const Thresholds th = vote_thresholds(prm, depth);
    const uint32_t vt = th.vt, it = th.it;
    Tally t{0, 0, -1, 0};
    tally(t, cA, vt, it, 0, 0);
    tally(t, cC, vt, it, 1, 0);
    tally(t, cG, vt, it, 2, 0);
    tally(t, cT, vt, it, 3, 0);
    if (cDel) tally(t, cDel, vt, it, 4, 0);                  // "-" exists only if it was seen (a HashMap entry)
    if (matched) tally(t, matched, vt, it, 5, 0);            // the 1-char string of a non-ACGT draft base
    if (n_other) t = tally_others(oc, pos, vt, it, t);
    PosOut o;
    o.rec = 0;
    o.packed = (orig == '-' ? 0u : 1u) | (orig << 16);
    uint32_t status;                                          // 0 low_depth 1 none 2 multiple 3 too_close 4 kept 5 changed
    if (th.low) status = 0;
    else if (t.nvalid == 0) status = 1;
    else if (t.nvalid > 1) status = 2;
    else if (t.ninter > 0) status = 3;
    else {
        status = 4;
        if (t.which <= 3) {
            const uint32_t nb = (uint32_t)"ACGT"[t.which];
            if (nb != orig) status = 5;
            o.packed = 1u | (nb << 16) | (nb != orig ? 1u << 24 : 0u);
        } else if (t.which == 4) {
            if (orig != '-') status = 5;
            o.packed = 0u | ((uint32_t)'-' << 16) | (orig != '-' ? 1u << 24 : 0u);
        } else if (t.which == 6) {
            const uint32_t len = (uint32_t)oc.nodes[t.rec].val & 0xFFFFu;
            uint32_t n = 0;
            for (uint32_t q = 0; q < len; ++q) n += other_char<BITS>(oc, t.rec, q) != '-';
            // an other-allele string never equals the draft's own 1-char string (those entries are "matched")
            status = 5;
            o.packed = (n & 0xFFFFu) | (1u << 24) | (1u << 25);
            o.rec = t.rec;
        }
    }
    o.packed |= status << 26;
    if (vp.dbg) debug_record(vp.dbg + pos, depth, vt, it, cA, cC, cG, cT, cDel, matched, n_other, orig, status, o);
    if (CHG && status == 5) {
        const uint32_t slot = atomicAdd(vp.chg_n, 1u);
        if (slot < vp.chg_cap) {
            vp.chg_pos[slot] = pos;
            debug_record(vp.chg + slot, depth, vt, it, cA, cC, cG, cT, cDel, matched, n_other, orig, status, o);
        }
    }
    return o;
}

// ------------------------------------------------------------------------------------------------------
// k_tile
// ------------------------------------------------------------------------------------------------------
#define TL_DN_HALO 32
#define TL_INV_K 32                                  // draft nibbles are staged for tile positions [-32, T + 32)
#define TL_DN_WORDS ((TL_T + 2 * TL_DN_HALO) / 16)

struct WalkStage {                                     // per warp: staging of the ordered-depth merge (depth_walk_two)
    uint4 ent[64];                                     // start, kept entries, 1/k (two words)
    uint32_t key[2][32];                               // alignment indices of the entries being merged, compacted, per run
};

// Per warp: one chunk of the chunk loop (32 consecutive slots) in shared memory, copied in by one bulk copy per array that
// completes on the stage's mbarrier.  Bases first: word 24 of lane 31's read, which the trim may load and then not use, is rec[0].
#define TL_STAGES 2
struct ChunkStage {
    uint4 seq[32 * TL_SEQ_QUADS];                      // 4-bit mode: the slots' bases (sseq)
    TileRec rec[32];                                   // the slots' records (srec)
};

#if defined(PP_EMULATE)
// The CPU emulator's strict model of the bulk copies and mbarriers (tests/emu/cuda_emu.h): a protocol error fails there.
static inline void stage_bar_init(unsigned long long* bar) { emu::ring_init(bar); }
static inline void stage_fence() {}
static inline void stage_expect(unsigned long long* bar, uint32_t bytes) { emu::ring_expect(bar, bytes); }
static inline void stage_copy(void* dst, const void* src, uint32_t bytes, unsigned long long* bar) { emu::ring_copy(dst, src, bytes, bar); }
static inline void stage_wait(unsigned long long* bar, uint32_t parity) { emu::ring_wait(bar, parity); }
#else
__device__ __forceinline__ uint32_t smem_addr(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void stage_bar_init(unsigned long long* bar) {   // one arrival per phase: the issuing lane's expect_tx
    asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;\n\tfence.mbarrier_init.release.cluster;" ::"r"(smem_addr(bar)) : "memory");
}
// Orders this thread's generic shared-memory writes before later bulk copies (async proxy) into the same bytes.
__device__ __forceinline__ void stage_fence() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
__device__ __forceinline__ void stage_expect(unsigned long long* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_addr(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void stage_copy(void* dst, const void* src, uint32_t bytes, unsigned long long* bar) {   // 16 B aligned, bytes % 16 == 0
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 ::"r"(smem_addr(dst)), "l"(src), "r"(bytes), "r"(smem_addr(bar)) : "memory");
}
__device__ __forceinline__ void stage_wait(unsigned long long* bar, uint32_t parity) {
    uint32_t done;
    do {
        asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
                     : "=r"(done) : "r"(smem_addr(bar)), "r"(parity) : "memory");
    } while (!done);
}
#endif

struct TileShared {
    int cdiff[TL_T + 4];                               // cover: +1 / -1 at interval ends, after the prefix sum = cover[p]
    uint32_t ex[4][TL_T];                              // A, C, G, T entries that differ from the draft base
    uint32_t del[TL_T];                                // "-" entries
    uint32_t oth[TL_T];                                // entries carrying any other allele (their distinct strings: the global chains)
    union {                                            // (per position both belong to the thread, then the warp, that votes on it)
        unsigned long long deficit[TL_T + 4];          // fixed-point depth deficit of k != 1 alignments (depth_bounds): +d / -d at
                                                       // interval ends, after the prefix sum the deficit of the position
        double depth[TL_T];                            // ordered f64 depth, written over the deficit in sub-tiles that walk
    };
    unsigned long long dn[TL_DN_WORDS + 2];            // 4-bit draft codes, 16 per word, position -32 first
    union {                                            // (phase D only, behind barriers | phase B)
        WalkStage wstage[TL_THREADS / 32];             // ordered-depth merge staging, one per warp
        ChunkStage ring[TL_THREADS / 32][TL_STAGES];   // chunk-loop stages, two per warp
    };
    unsigned long long ring_bar[TL_THREADS / 32][TL_STAGES];   // one mbarrier per stage
    uint2 queue[TL_QCAP];                              // (sorted slot, k) of the reads waiting for the general walk
    uint32_t qn;
    unsigned long long s_warp[TL_THREADS / 32];
    unsigned long long s_total;
    long long s_delta[TL_THREADS / 32];
    uint32_t tile;
    uint32_t any_multi;                                // an alignment with k != 1 touches the tile (the deficit is not all zero)
    double inv_k[TL_INV_K + 1];                        // 1.0 / k for small k (the ordered-depth walk divides once per slot otherwise)
    unsigned long long def_k[TL_INV_K + 1];            // depth_deficit(k) for small k (add_interval divides otherwise)
};
static_assert(sizeof(TileShared) <= 232448, "k_tile's shared memory: at most 227 KB per CTA on sm_90");

template <int BITS> struct TileCtx {
    const DevData& d;
    TileShared& sh;
    uint32_t P0;                                       // first position of the tile

    __device__ __forceinline__ bool in_tile(uint32_t pos) const { return pos - P0 < (uint32_t)TL_T; }
    __device__ __forceinline__ uint32_t draft_sym(uint32_t pos) const {        // pos inside the tile (+- halo)
        if (BITS == 4) {
            const uint32_t o = pos - P0 + TL_DN_HALO;
            return (uint32_t)(sh.dn[o >> 4] >> ((o & 15) * 4)) & 15u;
        }
        const uint32_t b = d.draft[pos];
        return b == '-' ? 0u : b;                       // a '-' in the draft never "matches" a read base: both count as "-"
    }
    __device__ __forceinline__ void push_other(uint32_t pos, unsigned long long aln, uint32_t start, uint32_t len, unsigned long long sig) {
        if (!in_tile(pos)) return;
        atomicAdd(&sh.oth[pos - P0], 1u);               // entries (not distinct alleles): feeds `matched`
        other_insert<BITS>(d, pos, (aln << 32) | ((unsigned long long)(start & 0xFFFFu) << 16) | (len & 0xFFFFu), sig);
    }
    // one single-base entry at reference position pos carrying read symbol s (read index ri)
    __device__ __forceinline__ void count_base(uint32_t pos, uint32_t s, unsigned long long aln, uint32_t ri) {
        if (!in_tile(pos)) return;
        if (Seq<BITS>::is_del(s)) { atomicAdd(&sh.del[pos - P0], 1u); return; }
        const uint32_t ds = draft_sym(pos);
        if (s == ds) return;                                   // counted implicitly: cover - explicit
        const int c = Seq<BITS>::acgt(s);
        if (c >= 0) atomicAdd(&sh.ex[c][pos - P0], 1u);
        else push_other(pos, aln, ri, 1, 1ull | ((unsigned long long)s << (BITS == 4 ? 4 : 8)));
    }
    // an alignment of a read with k good alignments keeps entries [gstart, gstart + nkept): interval add restricted to the tile
    __device__ __forceinline__ void add_interval(uint32_t gstart, uint32_t nkept, uint32_t k) {
        const long long a64 = (long long)gstart - (long long)P0, b64 = a64 + (long long)nkept;
        const int a = (int)max(a64, 0ll), b = (int)min(b64, (long long)TL_T);
        if (b <= a) return;
        atomicAdd(&sh.cdiff[a], 1); atomicAdd(&sh.cdiff[b], -1);
        if (k != 1) {
            const unsigned long long dk = k <= (uint32_t)TL_INV_K ? sh.def_k[k] : depth_deficit(k);
            atomicAdd(&sh.deficit[a], dk); atomicAdd(&sh.deficit[b], 0ull - dk);
            sh.any_multi = 1u;
        }
    }
    // 32 draft codes for tile-relative positions [rel0, rel0 + 32), rel0 in (-32, T)
    __device__ __forceinline__ void draft32(int rel0, unsigned long long& d0, unsigned long long& d1) const {
        load_nib32(sh.dn, (uint32_t)(rel0 + TL_DN_HALO), d0, d1);
    }
    // 4-bit only: `vc` (<= 32) single-base entries whose read codes are the low nibbles of r0:r1, at reference
    // positions pos0.. ; ri0 = read index of the first one.  One explicit count per in-tile base that differs from the draft.
    __device__ __forceinline__ void scan_mismatches(unsigned long long r0, unsigned long long r1, uint32_t vc, uint32_t pos0,
                                                    unsigned long long aln, uint32_t ri0) {
        const long long rel64 = (long long)pos0 - (long long)P0;
        if (rel64 <= -32 || rel64 >= (long long)TL_T) return;
        const int rel0 = (int)rel64;
        unsigned long long d0, d1;
        draft32(rel0, d0, d1);
        unsigned long long m0, m1;
        mismatch_masks(r0, r1, d0, d1, vc, m0, m1);
        // keep nibbles n with 0 <= rel0 + n < T
        const int lo = -rel0, hi = TL_T - rel0;              // valid n in [lo, hi)
        m0 &= nibmask(hi) & ~nibmask(lo);
        m1 &= nibmask(hi - 16) & ~nibmask(lo - 16);
        while (m0) {
            const uint32_t j = (uint32_t)(__ffsll((long long)m0) - 1) >> 2;
            m0 &= m0 - 1;
            const uint32_t code = (uint32_t)(r0 >> (4 * j)) & 15u;
            const int c = Seq<4>::acgt(code);
            if (c >= 0) atomicAdd(&sh.ex[c][rel0 + (int)j], 1u);
            else push_other(pos0 + j, aln, ri0 + j, 1, 1ull | ((unsigned long long)code << 4));
        }
        while (m1) {
            const uint32_t j = (uint32_t)(__ffsll((long long)m1) - 1) >> 2;
            m1 &= m1 - 1;
            const uint32_t code = (uint32_t)(r1 >> (4 * j)) & 15u;
            const int c = Seq<4>::acgt(code);
            if (c >= 0) atomicAdd(&sh.ex[c][rel0 + 16 + (int)j], 1u);
            else push_other(pos0 + 16 + j, aln, ri0 + 16 + j, 1, 1ull | ((unsigned long long)code << 4));
        }
    }
};

// Where the general walk reads a read's bases, by effective read index (reverse complement applied): sym(i) = base i, read32(ri)
// = the codes of bases [ri, ri + 32) (4-bit only; bases at indices >= len come out as garbage, the caller masks them).
// PoolBases: the stored read in the pool, reverse complemented on the fly - the queue, the long list and the 8-bit pool.
template <int BITS> struct PoolBases {
    const uint8_t* p;
    uint32_t len;
    bool rc;
    __device__ __forceinline__ PoolBases(const DevData& d, const TileRec& r)
        : p(d.seq_pool + (size_t)r.seq_off * (BITS == 4 ? 16 : 32)), len(r.len_nc & 0xFFFFu), rc(r.flags & TR_RC) {}
    __device__ __forceinline__ PoolBases(const DevData& d, unsigned long long aln)      // (alignment aln in SAM order)
        : p(d.seq_pool + (size_t)d.seq_off[aln] * (BITS == 4 ? 16 : 32)), len(d.seq_len[aln]), rc(d.flags[aln] & PP_FLAG_RC) {}
    __device__ __forceinline__ uint32_t sym(uint32_t i) const { return Seq<BITS>::read_sym(p, 0, len, rc, i); }
    __device__ __forceinline__ void read32(uint32_t ri, unsigned long long& r0, unsigned long long& r1) const {
        load_read32(reinterpret_cast<const unsigned long long*>(p), len, rc, ri, r0, r1);
    }
};
// StagedBases: a TR_STAGED slot's copy in the chunk ring (k_permute_seq: forward, base i = nibble i of its 24 words).  A window
// reads up to 4 words past the last base: the next slot's copy, or for lane 31 the first record of the stage (ChunkStage).
struct StagedBases {
    const uint32_t* w;
    __device__ __forceinline__ uint32_t sym(uint32_t i) const { return (w[i >> 3] >> ((i & 7) * 4)) & 15u; }
    __device__ __forceinline__ void read32(uint32_t ri, unsigned long long& r0, unsigned long long& r1) const {
        const uint32_t* q = w + (ri >> 3);
        const uint32_t sh = (ri & 7) * 4, x0 = q[0], x1 = q[1], x2 = q[2], x3 = q[3], x4 = q[4];
        r0 = (unsigned long long)__funnelshift_r(x0, x1, sh) | (unsigned long long)__funnelshift_r(x1, x2, sh) << 32;
        r1 = (unsigned long long)__funnelshift_r(x2, x3, sh) | (unsigned long long)__funnelshift_r(x3, x4, sh) << 32;
    }
};

// The entries of an alignment with E entries that survive the homopolymer trim (alignment.rs:364-378): walk the entries from the
// right, stop at the first one that is not the single base `last`, and drop that one too.  The CIGAR holds only M = X I D and
// consumes exactly `len` >= 1 read bases.
template <class Bases>
__device__ __forceinline__ unsigned long long kept_entries(const uint32_t* ops, uint32_t ncig, uint32_t len, unsigned long long E, const Bases& bs) {
    const uint32_t last = bs.sym(len - 1);
    unsigned long long run = 0;
    uint32_t ri = len;            // read index just past the current entry's M-part
    uint32_t pend = 0;            // inserted bases that extend the entry being visited
    bool stop = false;
    for (int p = (int)ncig - 1; p >= 0 && !stop; --p) {
        const uint32_t op = ops[p], o = op & 15u, l = op >> 4;
        if (o == PP_OP_I) { pend += l; ri -= l; continue; }
        if (o == PP_OP_D) {
            // entries (ri, ri + pend): only the rightmost can carry pend; equal to `last` iff pend == 1 and base == last
            for (uint32_t t = 0; t < l; ++t) {
                if (pend == 1 && bs.sym(ri) == last) { run++; pend = 0; }
                else { stop = true; break; }
            }
            continue;
        }
        for (uint32_t t = 0; t < l; ++t) {                    // M / = / X
            if (pend == 0 && bs.sym(ri - 1) == last) { run++; ri--; }
            else { stop = true; break; }
        }
    }
    return (E - run >= 1) ? (E - run - 1) : 0;
}

// Once per dataset, after the sequence pool has arrived and only when k_bin left any ERR_PAST_END: an alignment that starts at or
// past its contig's end is an overrun if the trim keeps an entry; if it keeps none the reference never indexes the pileup, so it
// is a good alignment that adds nothing (k_goodk counts it in `used` and in its read group's k; its key is already "nothing").
// The bases are the record's own or, for SEQ="*", its group's (seq_off / PP_FLAG_RC as the packers set them).
template <int BITS>
__device__ __forceinline__ void past_end_body(const DevData& d) {
    for (unsigned long long aln = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x; aln < d.n_aln; aln += (unsigned long long)gridDim.x * blockDim.x) {
        const uint32_t q = d.gq[aln];
        if (((q >> 5) & 7u) != ERR_PAST_END) continue;
        const uint32_t ncig = d.n_cigar[aln], len = d.seq_len[aln];
        const uint32_t* ops = d.cigar_ops + d.cigar_off[aln];
        unsigned long long E = 0;
        for (uint32_t p = 0; p < ncig; ++p)
            if ((ops[p] & 15u) != PP_OP_I) E += ops[p] >> 4;  // M, =, X, D (k_bin checked the ops and the length)
        const uint32_t err = (len != 0 && kept_entries(ops, ncig, len, E, PoolBases<BITS>(d, aln)) != 0) ? ERR_OOB : 0u;
        d.errc[aln] = (uint8_t)err;
        d.gq[aln] = (uint16_t)((q & ~(7u << 5)) | (err << 5));
    }
}
#if !defined(PP_EMULATE)
template <int BITS> __global__ void __launch_bounds__(256) k_past_end(DevData d) { past_end_body<BITS>(d); }
#endif

// The general CIGAR walk of one alignment (alignment.rs:175-201, 364-378; pileup.rs:189-200), restricted to the tile, reading the
// bases from `bs`.  Returns the number of kept entries.
template <int BITS, class Bases>
__device__ uint32_t general_walk(TileCtx<BITS>& S, const TileRec& r, uint32_t k, const Bases bs) {
    const DevData& d = S.d;
    const unsigned long long aln = r.aln;
    const uint32_t len = r.len_nc & 0xFFFFu, ncig = r.len_nc >> 16;
    const uint32_t gstart = r.gstart;
    const uint32_t* ops = d.cigar_ops + r.cigar_off;
    unsigned long long E = r.E;                                 // (k_bin's count, exact below its saturation)
    if (r.E == 0xFFFFFFFFu) {
        E = 0;
        for (uint32_t p = 0; p < ncig; ++p) {
            const uint32_t op = ops[p], o = op & 15u, l = op >> 4;
            if (o != PP_OP_I) E += l;                           // M, =, X, D (k_bin rejected everything else)
        }
    }
    const unsigned long long nk64 = kept_entries(ops, ncig, len, E, bs);
    if ((unsigned long long)gstart + nk64 > r.cend) { report_error(d.st, aln, ERR_OOB); return 0; }
    const uint32_t nkept = (uint32_t)nk64;
    S.add_interval(gstart, nkept, k);
    // positions of this tile the alignment can touch: entries [e_lo, e_hi)
    const long long off = (long long)S.P0 - (long long)gstart;
    const unsigned long long e_lo = off > 0 ? (unsigned long long)off : 0ull;
    const unsigned long long e_hi = min((unsigned long long)nkept, (unsigned long long)max(off + (long long)TL_T, 0ll));
    if (e_lo >= e_hi) return nkept;
    // emit entries e < nkept
    unsigned long long e = 0;
    uint32_t ri = 0;
    for (uint32_t p = 0; p < ncig && e < e_hi; ++p) {
        const uint32_t op = ops[p], o = op & 15u, l = op >> 4;
        if (o == PP_OP_I) { ri += l; continue; }
        uint32_t ins = 0;                                     // inserted bases right after this op
        for (uint32_t q = p + 1; q < ncig && (ops[q] & 15u) == PP_OP_I; ++q) ins += ops[q] >> 4;
        const unsigned long long plain64 = min((unsigned long long)(ins ? l - 1 : l), (unsigned long long)nkept - e);   // plain single entries of this op that are kept
        // the part of [e, e + plain64) inside the tile
        const unsigned long long t_lo = e_lo > e ? e_lo - e : 0ull, t_hi = min(plain64, e_hi > e ? e_hi - e : 0ull);
        if (o == PP_OP_D) {
            for (unsigned long long t = t_lo; t < t_hi; ++t) atomicAdd(&S.sh.del[(uint32_t)(gstart + e + t) - S.P0], 1u);
            if (ins && e + l - 1 < nkept) {                   // the last "-" entry absorbs a following insertion
                const uint32_t pos = (uint32_t)(gstart + e + l - 1);
                if (ins == 1) S.count_base(pos, bs.sym(ri), aln, ri);
                else S.push_other(pos, aln, ri, ins, make_sig<BITS>(bs, ri, ins));
            }
            e += l;
            continue;
        }
        if (BITS == 4) {
            for (unsigned long long c0 = t_lo & ~31ull; c0 < t_hi; c0 += 32) {
                unsigned long long r0, r1;
                bs.read32(ri + (uint32_t)c0, r0, r1);
                S.scan_mismatches(r0, r1, (uint32_t)min(plain64 - c0, 32ull), (uint32_t)(gstart + e + c0), aln, ri + (uint32_t)c0);
            }
        } else {
            for (unsigned long long t = t_lo; t < t_hi; ++t)
                S.count_base((uint32_t)(gstart + e + t), bs.sym(ri + (uint32_t)t), aln, ri + (uint32_t)t);
        }
        if (ins && e + l - 1 < nkept)
            S.push_other((uint32_t)(gstart + e + l - 1), aln, ri + l - 1, 1 + ins, make_sig<BITS>(bs, ri + l - 1, 1 + ins));
        e += l;
        ri += l;
    }
    return nkept;
}

// The fast path: a 4-bit read of at most 192 bases whose CIGAR is one M / = run, or two of them around one insertion or deletion
// (TR_FAST1: aM bI cM / aM bD cM).  Its bases were copied into slot order when the dataset was binned - forward strand, base i =
// nibble i (k_permute_seq) - so slot i's read is the 96 bytes at sseq + 6 i, next to its neighbours' in the tile's list: a warp's 32
// reads are 3 KB of consecutive memory, which the chunk loop copies into shared memory with one bulk copy.  `w` = the read's 24 words
// (shared memory; word 24 may be read and is then not used).  The draft comes from the tile's shared-memory copy through one native
// funnel shift per 8 bases.  The read's single-base entries are at most two segments of the read, each at its own draft offset: A =
// the first match run, B = the last one of a one-indel read (empty for a plain read).
//   pass 1: XOR against the draft four words at a time and only record WHICH words differ - straight-line code, no divergence.  A
//           group of four words compares at segment A's offset if it holds a whole word of A, else at B's;
//   pass 2: the edge words (partly outside a segment or the tile: among them the words at the boundary and those with inserted
//           bases), the whole words of B in a group compared at A's offset, and the few words that differ (about one word in two
//           reads) are loaded again and every differing base is counted, once per segment the word holds.
// Only the insertion's allele, the deletion's "-" entries and pass 2 diverge between plain and one-indel reads.
// Returns kept entries, or NONE32 = "take the general walk" (a homopolymer tail of 8+ bases or one longer than the last match run, a
// read shorter than 8).
__device__ __forceinline__ uint32_t fast_walk(TileCtx<4>& S, const TileRec& r, const uint32_t* w, uint32_t k) {
    const uint32_t len = r.len_nc & 0xFFFFu;
    const unsigned long long aln = r.aln;
    if (len < 8) return NONE32;
    // ---- trim (alignment.rs:364-378): how many of the last bases equal the last one.  The last 8 bases as one word.
    uint32_t run;
    const uint32_t tw = (len - 8) >> 3;                          // the two words the trim looks at: tw, tw + 1
    const uint32_t tw0 = w[tw], tw1 = w[tw + 1];
    {
        const uint32_t o = len - 8;
        const uint32_t t8 = __funnelshift_r(tw0, tw1, (o & 7) * 4);
        const uint32_t x = t8 ^ ((t8 >> 28) * 0x11111111u);
        const uint32_t nz = (x | (x >> 1) | (x >> 2) | (x >> 3)) & 0x11111111u;
        if (nz == 0) return NONE32;                            // 8+ equal bases at the end: the general walk counts them
        run = 7u - ((31u - (uint32_t)__clz((int)nz)) >> 2);
    }
    const bool one = r.flags & TR_FAST1;
    const uint32_t ia = (r.flags >> 8) & 0xFFu, ib = (r.flags >> 16) & 0xFFFu;            // (0 for a plain read)
    const bool is_del = (r.flags >> 28) & 1u;
    // The general walk's trim stops at the start of the last match run: before it, a D entry carries no inserted base (its `pend` is
    // 0, so it never counts) and the entry before an I carries the inserted bases (pend != 0).  So the trim is `run` while run <= lc;
    // beyond that the 8-base window has looked past the run, and the general walk takes the read.  (A plain read: lc = len >= 8 > run.)
    const uint32_t lc = len - ia - (is_del ? 0u : ib);
    if (run > lc) return NONE32;
    const uint32_t E = is_del ? len + ib : len - ib;
    const uint32_t nkept = E - run - 1;                         // >= a - 1 (I) / a + b - 1 (D): segment A is always kept whole
    if ((unsigned long long)r.gstart + nkept > r.cend) { report_error(S.d.st, aln, ERR_OOB); return 0; }
    S.add_interval(r.gstart, nkept, k);
    const long long g0 = (long long)r.gstart - (long long)S.P0;
    if (g0 >= (long long)TL_T || g0 + (long long)nkept <= 0) return nkept;
    const uint32_t* dn32 = reinterpret_cast<const uint32_t*>(S.sh.dn);
    // Segment s: read bases [lo, hi) are single-base entries at tile-relative positions relq + base, clipped to the tile.
    //   plain: A = [0, nkept);  aM bI cM: A = [0, a - 1), entry a - 1 carries 1 + b bases (an "other" allele), B = [a + b, nkept + b) at
    //   relq - b;  aM bD cM: A = [0, a), b "-" entries, B = [a, nkept - b) at relq + b.
    int relq[2], lo[2], hi[2], i0[2];
    uint32_t sh4[2], inner[2], edge[2];
    relq[0] = (int)g0;
    relq[1] = (int)g0 + (is_del ? (int)ib : -(int)ib);
    lo[0] = 0;
    hi[0] = !one ? (int)nkept : (int)ia - (is_del ? 0 : 1);
    lo[1] = one ? (int)(ia + (is_del ? 0u : ib)) : 0;
    hi[1] = one ? (int)nkept + (is_del ? -(int)ib : (int)ib) : 0;
#pragma unroll
    for (int s = 0; s < 2; ++s) {
        lo[s] = max(lo[s], -relq[s]);
        hi[s] = min(hi[s], (int)TL_T - relq[s]);
        const int o0 = relq[s] + TL_DN_HALO;                   // nibble offset of word 0 in the staged draft
        i0[s] = o0 >> 3;                                        // floor; i0 + m >= 0 for every word of a group that holds a valid word
        sh4[s] = (uint32_t)(o0 & 7) * 4;
        inner[s] = edge[s] = 0;
        if (hi[s] > lo[s]) {
            const uint32_t first = (uint32_t)lo[s], lastn = (uint32_t)(hi[s] - 1), m_first = first >> 3, m_last = lastn >> 3;
            // an edge word needs its own visit only when it is partly outside [first, lastn] (a read that starts inside the tile starts
            // on a word boundary: its first word is a whole word like any other)
            edge[s] = ((first & 7) ? 1u << m_first : 0u) | ((lastn & 7) != 7 ? 1u << m_last : 0u);
            inner[s] = ((2u << m_last) - (1u << m_first)) & ~edge[s];
        }
    }
    uint32_t bits = 0, cmp = 0;                                 // cmp: the whole words pass 1 compared at their own segment's offset
#pragma unroll
    for (int g = 0; g < TL_SEQ_QUADS; ++g) {
        const uint32_t ga = (inner[0] >> (4 * g)) & 15u, gb = (inner[1] >> (4 * g)) & 15u;
        if (ga | gb) {
            const int j = (ga ? i0[0] : i0[1]) + 4 * g;
            const uint32_t sh = ga ? sh4[0] : sh4[1];
            const uint4 q = reinterpret_cast<const uint4*>(w)[g];
            const uint32_t d0 = dn32[j], d1 = dn32[j + 1], d2 = dn32[j + 2], d3 = dn32[j + 3], d4 = dn32[j + 4];
            if (q.x != __funnelshift_r(d0, d1, sh)) bits |= 1u << (4 * g);
            if (q.y != __funnelshift_r(d1, d2, sh)) bits |= 2u << (4 * g);
            if (q.z != __funnelshift_r(d2, d3, sh)) bits |= 4u << (4 * g);
            if (q.w != __funnelshift_r(d3, d4, sh)) bits |= 8u << (4 * g);
            cmp |= (ga ? ga : gb) << (4 * g);
        }
    }
    // every base of word m (value wv) that differs from the draft inside segment s
    auto count_word = [&](int s, uint32_t m, uint32_t wv) {
        const int sl0 = s ? lo[1] : lo[0], sh0 = s ? hi[1] : hi[0], rq = s ? relq[1] : relq[0];
        const int a = sl0 - 8 * (int)m, b = sh0 - 8 * (int)m;                     // the segment's nibbles of the word: [a, b)
        if (b <= 0 || a >= 8 || b <= a) return;
        const int j = (s ? i0[1] : i0[0]) + (int)m;
        uint32_t x = wv ^ __funnelshift_r(dn32[j], dn32[j + 1], s ? sh4[1] : sh4[0]);
        if (a > 0) x &= 0xFFFFFFFFu << (4 * a);
        if (b < 8) x &= 0xFFFFFFFFu >> (32 - 4 * b);
        uint32_t nz = (x | (x >> 1) | (x >> 2) | (x >> 3)) & 0x11111111u;
        while (nz) {
            const uint32_t t = (uint32_t)(__ffs((int)nz) - 1) >> 2;
            nz &= nz - 1;
            const uint32_t code = (wv >> (4 * t)) & 15u;
            const int rel = rq + 8 * (int)m + (int)t;
            if ((code & (code - 1)) == 0) atomicAdd(&S.sh.ex[__ffs((int)code) - 1][rel], 1u);      // A, C, G, T = 1, 2, 4, 8
            else S.push_other(S.P0 + (uint32_t)rel, aln, 8u * m + t, 1, 1ull | ((unsigned long long)code << 4));
        }
    };
    uint32_t mm = (bits & cmp) | ((inner[0] | inner[1]) & ~cmp) | edge[0] | edge[1];
    // the partial last word of a read that ends inside the tile is one of the two words the trim already holds: straight-line (when
    // it is not also a word of segment A before a boundary)
    {
        const bool sb = hi[1] > lo[1];                         // the segment that ends the read's kept entries
        const int e_lo = sb ? lo[1] : lo[0], e_hi = sb ? hi[1] : hi[0];
        const uint32_t m_last = (uint32_t)(e_hi - 1) >> 3;
        if (e_hi > e_lo && (((sb ? edge[1] : edge[0]) >> m_last) & 1u) && m_last - tw < 2u && (!sb || hi[0] <= 8 * (int)m_last)) {
            mm &= ~(1u << m_last);
            count_word(sb ? 1 : 0, m_last, m_last == tw ? tw0 : tw1);
        }
    }
    while (mm) {                                               // words that differ (about one word in two reads), edge words
        const uint32_t m = (uint32_t)__ffs((int)mm) - 1;
        mm &= mm - 1;
        const uint32_t wv = w[m];
        count_word(0, m, wv);
        if (one) count_word(1, m, wv);
    }
    if (one) {
        if (!is_del) {
            if (ia - 1 < nkept)
                S.push_other(r.gstart + ia - 1, aln, ia - 1, 1 + ib, make_sig<4>(StagedBases{w}, ia - 1, 1 + ib));
        } else {
            const long long t0 = g0 + (long long)ia;             // the kept "-" entries: [a, min(a + b, nkept))
            const long long t_lo = max(0ll, -t0), t_hi = min((long long)min(ib, nkept - ia), (long long)TL_T - t0);
            for (long long t = t_lo; t < t_hi; ++t) atomicAdd(&S.sh.del[(int)(t0 + t)], 1u);
        }
    }
    return nkept;
}

// The record of sorted slot i (coalesced: consecutive lanes, consecutive 32-byte records).
__device__ __forceinline__ TileRec load_srec(const DevData& d, uint32_t slot) {
    const uint4* src = reinterpret_cast<const uint4*>(d.srec + slot);
    const uint4 a = __ldg(src), b = __ldg(src + 1);
    TileRec r;
    r.gstart = a.x; r.seq_off = a.y; r.cigar_off = a.z; r.len_nc = a.w; r.aln = b.x; r.E = b.y; r.flags = b.z; r.cend = b.w;
    return r;
}

// The ordered depth of one 128-position sub-tile (pileup.rs:64 in SAM order).  The alignments that can cover it live in up to
// DW_RUNS runs of the sorted list - the bins that can reach it and the long list - each of them in SAM order.  One warp merges
// the runs by alignment index: a window of 32 slots per run sits in registers (one coalesced 16-byte load per lane, the next
// window prefetched), entries that do not overlap the sub-tile are skipped through a ballot mask, and 1/k is added with
// round-to-nearest in merged (= SAM) order, four consecutive positions per lane.
#define DW_RUNS 4
#if defined(PP_EMULATE)
#define PP_PREFETCH_L1(p) ((void)(p))
#define PP_PREFETCH_L2(p) ((void)(p))
#else
#define PP_PREFETCH_L1(p) asm volatile("prefetch.global.L1 [%0];" ::"l"(p))
#define PP_PREFETCH_L2(p) asm volatile("prefetch.global.L2 [%0];" ::"l"(p))
#endif
template <int BITS>
__device__ void depth_walk_steps(const DevData& d, TileShared& sh, uint32_t P0, uint32_t sub, uint32_t lb, uint32_t long_lo, uint32_t long_hi) {
    const uint32_t lane = threadIdx.x & 31;
    const uint32_t s = P0 + sub * PP_SUB;
    const uint32_t bin = s >> PP_BIN_SHIFT;
    uint32_t wb[DW_RUNS], end[DW_RUNS], mask[DW_RUNS], head[DW_RUNS];
    uint32_t w_aln[DW_RUNS], w_start[DW_RUNS], w_len[DW_RUNS];
    double w_inv[DW_RUNS];
    // window of run r at slot wb[r]; windows without an overlapping entry are skipped
    auto load_window = [&](int r) {
        for (;;) {
            if (wb[r] >= end[r]) { mask[r] = 0; head[r] = NONE32; return; }
            const uint32_t slot = wb[r] + lane;
            uint4 q = make_uint4(NONE32, 0, 0, 1);
            if (slot < end[r]) {
                q = d.wrec[slot];
                if (slot + 32 < end[r]) PP_PREFETCH_L1(d.wrec + slot + 32);
            }
            uint32_t len = q.z;
            if (r == DW_RUNS - 1 && slot < end[r]) {            // long list: this CTA walked the alignment only if it can touch the tile
                const TileRec rec = load_srec(d, slot);
                const unsigned long long e_end = (unsigned long long)rec.gstart + rec.E;
                const uint32_t kk = d.kf[rec.aln];
                // this CTA wrote the slot only if the alignment contributes and can touch the tile
                const bool mine = kk != 0 && e_end > P0 && rec.gstart < P0 + (uint32_t)TL_T;
                q.x = rec.aln; q.y = rec.gstart; q.w = mine ? kk : 1u;
                len = mine ? q.z : 0u;
            }
            const bool ov = slot < end[r] && len != 0 && q.y < s + PP_SUB && q.y + len > s;
            const uint32_t m = __ballot_sync(0xffffffffu, ov);
            w_aln[r] = q.x; w_start[r] = q.y; w_len[r] = len;
            w_inv[r] = q.w <= (uint32_t)TL_INV_K ? sh.inv_k[q.w] : __ddiv_rn(1.0, (double)q.w);             // 1.0 / good_alignments.len() as f64 (alignment.rs:288)
            if (m) { mask[r] = m; head[r] = __shfl_sync(0xffffffffu, w_aln[r], __ffs((int)m) - 1); return; }
            wb[r] += 32;
        }
    };
#pragma unroll
    for (int r = 0; r < DW_RUNS; ++r) {
        wb[r] = end[r] = 0;
        if (r < DW_RUNS - 1) {
            if ((uint32_t)r <= lb && bin + (uint32_t)r >= lb) {
                const uint32_t b = bin + (uint32_t)r - lb;
                wb[r] = d.bin_start[b]; end[r] = d.bin_start[b + 1];
            }
        } else { wb[r] = long_lo; end[r] = long_hi; }
        w_aln[r] = NONE32; w_start[r] = 0; w_len[r] = 0; w_inv[r] = 0.0;
        load_window(r);
    }
    const uint32_t p = s + lane * 4;
    double dep0 = 0.0, dep1 = 0.0, dep2 = 0.0, dep3 = 0.0;
    for (;;) {
        uint32_t best = NONE32;
        int rb = -1;
#pragma unroll
        for (int r = 0; r < DW_RUNS; ++r) if (head[r] < best) { best = head[r]; rb = r; }
        if (rb < 0) break;
        uint32_t st = 0, ln = 0;
        double inv = 0.0;
#pragma unroll
        for (int r = 0; r < DW_RUNS; ++r) {
            if (r == rb) {                                      // warp-uniform
                const int src = __ffs((int)mask[r]) - 1;
                st = __shfl_sync(0xffffffffu, w_start[r], src);
                ln = __shfl_sync(0xffffffffu, w_len[r], src);
                inv = __shfl_sync(0xffffffffu, w_inv[r], src);
                mask[r] &= mask[r] - 1;
                if (mask[r]) head[r] = __shfl_sync(0xffffffffu, w_aln[r], __ffs((int)mask[r]) - 1);
                else { wb[r] += 32; load_window(r); }
            }
        }
        const uint32_t off = p - st;                            // position p + q is covered iff (off + q) < length (unsigned)
        if (off < ln) dep0 = __dadd_rn(dep0, inv);
        if (off + 1u < ln) dep1 = __dadd_rn(dep1, inv);
        if (off + 2u < ln) dep2 = __dadd_rn(dep2, inv);
        if (off + 3u < ln) dep3 = __dadd_rn(dep3, inv);
    }
    double* out = sh.depth + (p - P0);
    out[0] = dep0; out[1] = dep1; out[2] = dep2; out[3] = dep3;
}

// The same for the common case of at most two runs (reads of up to 256 entries, no long list): the merge is done 32 + 32 slots
// at a time - every lane ranks its own two entries against the other run's window by binary search in shared memory, the
// merged (start, length, 1/k) triples land in a per-warp staging area, and the ordered additions run over that area with
// nothing but broadcast loads in the loop.
template <int BITS>
__device__ void depth_walk_two(const DevData& d, TileShared& sh, WalkStage& ws, uint32_t P0, uint32_t sub, uint32_t lo0, uint32_t hi0, uint32_t lo1, uint32_t hi1) {
    const uint32_t lane = threadIdx.x & 31;
    const uint32_t s = P0 + sub * PP_SUB;
    const uint32_t lt = (1u << lane) - 1u;
    uint32_t wb[2] = {lo0, lo1}, end[2] = {hi0, hi1}, mask[2] = {0, 0}, lastkey[2] = {0, 0};
    uint32_t w_aln[2] = {NONE32, NONE32}, w_start[2] = {0, 0}, w_len[2] = {0, 0};
    double w_inv[2] = {0.0, 0.0};
    bool loaded[2] = {false, false};
    const uint32_t p = s + lane * 4;
    double dep0 = 0.0, dep1 = 0.0, dep2 = 0.0, dep3 = 0.0;
    for (;;) {
        // (re)load the windows that are used up; windows without an overlapping entry are skipped
#pragma unroll
        for (int r = 0; r < 2; ++r) {
            while (mask[r] == 0 && (!loaded[r] || wb[r] < end[r])) {
                if (loaded[r]) wb[r] += 32;
                loaded[r] = true;
                if (wb[r] >= end[r]) break;
                const uint32_t slot = wb[r] + lane;
                uint4 q = make_uint4(NONE32, 0, 0, 1);
                if (slot < end[r]) {
                    q = d.wrec[slot];
                    if (slot + 32 < end[r]) PP_PREFETCH_L2(d.wrec + slot + 32);    // (requesting the next window into registers instead was measured: no faster)
                }
                const bool ov = slot < end[r] && q.z != 0 && q.y < s + PP_SUB && q.y + q.z > s;
                mask[r] = __ballot_sync(0xffffffffu, ov);
                w_aln[r] = q.x; w_start[r] = q.y; w_len[r] = q.z;
                w_inv[r] = q.w <= (uint32_t)TL_INV_K ? sh.inv_k[q.w] : __ddiv_rn(1.0, (double)q.w);         // 1.0 / good_alignments.len() as f64 (alignment.rs:288)
                // every entry of the run up to this key is in this window or behind us; NONE32 once the run has no further window
                lastkey[r] = (wb[r] + 32 < end[r]) ? __shfl_sync(0xffffffffu, w_aln[r], 31) : NONE32;
            }
        }
        if ((mask[0] | mask[1]) == 0) break;                   // both runs exhausted
        // entries that can be merged now: alignment index <= the smaller "complete up to" key
        const uint32_t lim0 = (mask[0] || wb[0] < end[0]) ? lastkey[0] : NONE32, lim1 = (mask[1] || wb[1] < end[1]) ? lastkey[1] : NONE32;
        const uint32_t limit = min(lim0, lim1);
        uint32_t e[2], rank[2], n[2];
#pragma unroll
        for (int r = 0; r < 2; ++r) {
            e[r] = mask[r] & __ballot_sync(0xffffffffu, w_aln[r] <= limit);
            rank[r] = (uint32_t)__popc(e[r] & lt);
            n[r] = (uint32_t)__popc(e[r]);
            if ((e[r] >> lane) & 1u) ws.key[r][rank[r]] = w_aln[r];
        }
        __syncwarp();
#pragma unroll
        for (int r = 0; r < 2; ++r) {
            if ((e[r] >> lane) & 1u) {
                const uint32_t* ok = ws.key[r ^ 1];
                uint32_t blo = 0, bhi = n[r ^ 1];               // entries of the other run that come first
#pragma unroll
                for (int it = 0; it < 6; ++it) {
                    if (blo < bhi) { const uint32_t mid = (blo + bhi) >> 1; if (ok[mid] < w_aln[r]) blo = mid + 1; else bhi = mid; }
                }
                const unsigned long long iv = (unsigned long long)__double_as_longlong(w_inv[r]);
                ws.ent[rank[r] + blo] = make_uint4(w_start[r], w_len[r], (uint32_t)iv, (uint32_t)(iv >> 32));
            }
            mask[r] &= ~e[r];
        }
        __syncwarp();
        const uint32_t ntot = n[0] + n[1];
        for (uint32_t j = 0; j < ntot; ++j) {
            const uint4 q = ws.ent[j];
            const double inv = __longlong_as_double((long long)((unsigned long long)q.z | ((unsigned long long)q.w << 32)));
            const uint32_t off = p - q.x;                       // position p + i is covered iff (off + i) < length (unsigned)
            if (off < q.y) dep0 = __dadd_rn(dep0, inv);
            if (off + 1u < q.y) dep1 = __dadd_rn(dep1, inv);
            if (off + 2u < q.y) dep2 = __dadd_rn(dep2, inv);
            if (off + 3u < q.y) dep3 = __dadd_rn(dep3, inv);
        }
        __syncwarp();
    }
    double* out = sh.depth + (p - P0);
    out[0] = dep0; out[1] = dep1; out[2] = dep2; out[3] = dep3;
}

template <int BITS>
__device__ __forceinline__ void depth_walk(const DevData& d, TileShared& sh, WalkStage& ws, uint32_t P0, uint32_t sub, uint32_t lb, uint32_t long_lo, uint32_t long_hi) {
    const uint32_t bin = (P0 + sub * PP_SUB) >> PP_BIN_SHIFT;
    if (lb <= 1 && long_lo >= long_hi) {
        const uint32_t lo1 = d.bin_start[bin], hi1 = d.bin_start[bin + 1];
        uint32_t lo0 = 0, hi0 = 0;
        if (lb == 1 && bin >= 1) { lo0 = d.bin_start[bin - 1]; hi0 = lo1; }
        depth_walk_two<BITS>(d, sh, ws, P0, sub, lo0, hi0, lo1, hi1);
    } else depth_walk_steps<BITS>(d, sh, P0, sub, lb, long_lo, long_hi);
}

// CHG: the change report is recorded (vp.chg; without it the vp.chg* fields are not read).  A template argument, so that the kernel
// without the report does the work it did before the report existed (as a run-time test it measured up to 0.5 % slower on an H100,
// 700 W, 5 Mbp x 100x).
template <int BITS, bool CHG = false>
__device__ __forceinline__ void tile_body(const DevData& d, const VoteParams& vp, TileShared& sh) {
    const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const DevParams prm = *d.prm;
    const uint32_t lb = (d.max_ext + PP_BIN - 1) >> PP_BIN_SHIFT;               // bins a tile looks back (<= 2)
    const uint32_t long_lo = d.bin_start[d.n_bins], long_hi = d.bin_start[d.n_bins + 1];
    OthCtx oc;
    oc.nodes = d.nodes; oc.head = d.oth_head;
    oc.sr = SeqRef{d.seq_pool, d.seq_off, d.seq_len, d.flags};

    if (tid <= (uint32_t)TL_INV_K) {                                           // the same correctly rounded quotients, made once
        sh.inv_k[tid] = tid ? __ddiv_rn(1.0, (double)tid) : 0.0;
        sh.def_k[tid] = tid > 1 ? depth_deficit(tid) : 0ull;
    }
    ChunkStage* const ring = sh.ring[warp];
    unsigned long long* const bar = sh.ring_bar[warp];
    if (lane == 0) { stage_bar_init(&bar[0]); stage_bar_init(&bar[1]); }
    uint32_t parity = 0;                                                       // bit s: the phase stage s completes next (kept across tiles)
    for (;;) {
        // phase D's generic writes to the bytes the ring shares with `wstage` come before the next tile's bulk copies:
        // every thread fences its own writes, then the barrier
        stage_fence();
        __syncthreads();                                                       // everyone is done with the previous tile
        if (tid == 0) { sh.tile = atomicAdd(&d.st->ticket, 1u); sh.any_multi = 0; sh.qn = 0; }
        __syncthreads();
        if (sh.tile >= d.n_tiles) break;
        const uint32_t tile = d.tile_order[sh.tile];
        const uint32_t P0 = tile * (uint32_t)TL_T;
        TileCtx<BITS> S{d, sh, P0};
#ifdef PP_TILE_PROF
        long long pt[6];
        pt[0] = clock64();
#endif
        // The slots of the tile's bins and of the `lb` bins before it - one contiguous range of the binned dataset - and the first two
        // chunks' copies and SAM indices: a chain of dependent trips to memory (bin bounds, records, k words) that now runs under phase A.
        // (taking the next tile's ticket a tile early, to hide these trips, was measured: the greedy heaviest-first schedule then
        // looks one tile ahead and the kernel's tail grows)
        const uint32_t b0 = P0 >> PP_BIN_SHIFT;
        const uint32_t lo = d.bin_start[b0 >= lb ? b0 - lb : 0u];
        const uint32_t hi = d.bin_start[min(b0 + (uint32_t)(TL_T / PP_BIN), d.n_bins)];
        const uint32_t stride = 32u * (TL_THREADS / 32);
        uint32_t c_a = lo + 32u * warp;
        // lane 0: the records (and, 4-bit, the bases) of the chunk at slot c < hi into stage s; the last chunk of the range is shorter
        auto issue = [&](uint32_t c, uint32_t s) {
            const uint32_t n = min(32u, hi - c);
            stage_expect(&bar[s], n * (uint32_t)(sizeof(TileRec) + (BITS == 4 ? 16 * TL_SEQ_QUADS : 0)));
            stage_copy(ring[s].rec, d.srec + c, n * (uint32_t)sizeof(TileRec), &bar[s]);
            if (BITS == 4) stage_copy(ring[s].seq, d.sseq + (size_t)c * TL_SEQ_QUADS, n * 16u * TL_SEQ_QUADS, &bar[s]);
        };
        if (lane == 0) {
            if (c_a < hi) issue(c_a, 0);
            if (c_a + stride < hi) issue(c_a + stride, 1);
        }
        // Only two words per lane travel from one round of the chunk loop to the next - the SAM index of the NEXT chunk's record (what
        // its k word is gathered with) and that k word.  (Carrying whole records two chunks ahead cost 16 registers the fast walk does
        // not have: they lived on the stack, and every round began with their reloads from local memory.)
        const uint32_t last_slot = d.n_slots ? d.n_slots - 1 : 0u;
        uint32_t k_a = 0;
        const uint32_t aln_a = __ldg(&d.srec[min(c_a + lane, last_slot)].aln);
        uint32_t aln_b = __ldg(&d.srec[min(c_a + stride + lane, last_slot)].aln);
        // ---- phase A: clear the counters, stage the draft as 4-bit codes
        {
            uint4* z = reinterpret_cast<uint4*>(sh.cdiff);
            const uint32_t nz = (uint32_t)((size_t)((char*)sh.dn - (char*)sh.cdiff) / 16);   // cdiff, ex, del, oth, deficit
            for (uint32_t i = tid; i < nz; i += TL_THREADS) z[i] = make_uint4(0, 0, 0, 0);
            // ... and the tile's chain heads in HBM: only this tile's walks insert at its positions (push_other), so the 4 B per
            // position that a call has to zero are zeroed here, by the CTA that is about to use them, not by a memset over the assembly
            static_assert(TL_T == 4 * TL_THREADS, "one 16-byte store of chain heads per thread");
            reinterpret_cast<uint4*>(d.oth_head + P0)[tid] = make_uint4(0, 0, 0, 0);
            if (BITS == 4) {
                uint32_t* dn32w = reinterpret_cast<uint32_t*>(sh.dn);
                for (uint32_t wi = tid; wi < 2 * (TL_DN_WORDS + 2); wi += TL_THREADS) {      // 8 positions per 32-bit word
                    const long long g0 = (long long)P0 - TL_DN_HALO + 8ll * wi;
                    uint32_t v = 0;
                    if (g0 >= 0 && g0 + 8 <= (long long)d.G) {
                        const uint2 q = *reinterpret_cast<const uint2*>(d.draft + g0);       // draft is 16 B aligned, g0 a multiple of 8
#pragma unroll
                        for (int i = 0; i < 8; ++i) v |= asc2nib(((i < 4 ? q.x : q.y) >> ((i & 3) * 8)) & 255u) << (4 * i);
                    } else {
                        for (int i = 0; i < 8; ++i)
                            if (g0 + i >= 0 && g0 + i < (long long)d.G) v |= asc2nib(d.draft[g0 + i]) << (4 * i);
                    }
                    dn32w[wi] = v;
                }
            }
        }
        if (c_a + lane < hi) k_a = d.kf[aln_a];                // (the SAM index has arrived while the counters were cleared)
        __syncthreads();
#ifdef PP_TILE_PROF
        pt[1] = clock64();
#endif
        // ---- phase B: every alignment that can touch the tile: the slots of the tile's bins and of the `lb` bins before it - one
        // contiguous range of the binned dataset.  Warps take chunks of 32 consecutive slots round robin.  A chunk's records and bases
        // are 1 KB + 3 KB of consecutive memory: lane 0 copies them into one of the warp's two stages in shared memory one chunk ahead,
        // so the walk starts on data that is already there.  The only gather is the 4-byte "k / contributes" word of the current
        // options, fetched one chunk ahead.
        {
            // a TR_STAGED read the fast walk does not take (two or more indels, X ops, homopolymer tails of 8+ bases or longer than the
            // last match run, reads shorter than 8) is walked in place by the general walk, from its bases in the stage (only its
            // CIGAR ops come from memory).  What is left - reads longer than 192 bases, the 8-bit pool -
            // goes to a block-wide queue dealt to the warps after the chunk loop, each of its walks a chain of dependent loads
#ifdef PP_TILE_PROF
            unsigned long long wait_cyc = 0;
#endif
            uint32_t s = 0;                                    // the stage of chunk c_a
            while (c_a < hi) {
                const uint32_t c_b = c_a + stride, c_c = c_b + stride;
                // next chunk: its k word (its SAM index arrived during the previous round); the chunk after: its SAM index
                uint32_t k_b = 0;
                if (c_b + lane < hi) k_b = d.kf[aln_b];
                const uint32_t aln_c = __ldg(&d.srec[min(c_c + lane, last_slot)].aln);
#ifdef PP_TILE_PROF
                const long long w0 = clock64();
#endif
                stage_wait(&bar[s], (parity >> s) & 1u);
                parity ^= 1u << s;
#ifdef PP_TILE_PROF
                if (lane == 0) wait_cyc += (unsigned long long)(clock64() - w0);
#endif
                const TileRec rec_a = ring[s].rec[lane];      // (lanes past hi: bytes of an earlier chunk, not used)
                const uint32_t* const seq_a = reinterpret_cast<const uint32_t*>(ring[s].seq + lane * TL_SEQ_QUADS);
                const uint32_t i = c_a + lane;
                bool defer = false;
                if (i < hi) {
                    if (k_a == 0) d.wrec[i] = make_uint4(rec_a.aln, rec_a.gstart, 0u, 1u);           // adds nothing under these options
                    else {
                        uint32_t nk = NONE32;
                        if (BITS == 4 && (rec_a.flags & TR_FAST)) nk = fast_walk(reinterpret_cast<TileCtx<4>&>(S), rec_a, seq_a, k_a);
                        if (BITS == 4 && nk == NONE32 && (rec_a.flags & TR_STAGED))
                            nk = general_walk<4>(reinterpret_cast<TileCtx<4>&>(S), rec_a, k_a, StagedBases{seq_a});
                        if (nk == NONE32) defer = true;
                        else d.wrec[i] = make_uint4(rec_a.aln, rec_a.gstart, nk, k_a);
                    }
                }
                if (defer) {
#if defined(PP_EMULATE)
                    emu_n_queued.fetch_add(1, std::memory_order_relaxed);
#endif
                    const uint32_t qi = atomicAdd(&sh.qn, 1u);
                    if (qi < TL_QCAP) {
                        sh.queue[qi] = make_uint2(i, k_a);
                        PP_PREFETCH_L2(d.cigar_ops + rec_a.cigar_off);                  // what the general walk will chase
                        PP_PREFETCH_L2(d.seq_pool + (size_t)rec_a.seq_off * (BITS == 4 ? 16 : 32));
                    } else                                                             // (a tile with more than TL_QCAP such reads)
                        d.wrec[i] = make_uint4(rec_a.aln, rec_a.gstart, general_walk<BITS>(S, rec_a, k_a, PoolBases<BITS>(d, rec_a)), k_a);
                }
                __syncwarp();                                  // every lane is done with stage s: refill it with the chunk after next
                if (lane == 0 && c_c < hi) issue(c_c, s);
                c_a = c_b; aln_b = aln_c; k_a = k_b; s ^= 1u;
            }
#ifdef PP_TILE_PROF
            if (lane == 0 && wait_cyc) atomicAdd(&d.st->prof[11], wait_cyc);
#endif
        }
        __syncthreads();
#ifdef PP_TILE_PROF
        pt[2] = clock64();
#endif
        {
            // Each of these walks is a chain of dependent loads with its own branches: 32 of them on one warp run in lock step through
            // the union of their paths (measured: 38 queued reads per tile took a third of the tile's time on two warps).  So the
            // queue is dealt one read per WARP first - lane 0 of every warp, then lane 1, ... - and the walks overlap instead.
            const uint32_t qn = min(sh.qn, (uint32_t)TL_QCAP);
            for (uint32_t qi = lane * (TL_THREADS / 32) + warp; qi < qn; qi += TL_THREADS) {
                const uint2 q = sh.queue[qi];                   // (the entry carries k: the record is the only load before the walk)
                const TileRec r = load_srec(d, q.x);
                d.wrec[q.x] = make_uint4(r.aln, r.gstart, general_walk<BITS>(S, r, q.y, PoolBases<BITS>(d, r)), q.y);
            }
            // the long list: alignments of more than TL_LONG_E entries, looked at by every tile
            for (uint32_t i = long_lo + tid; i < long_hi; i += TL_THREADS) {
                const TileRec r = load_srec(d, i);
                const unsigned long long e_end = (unsigned long long)r.gstart + r.E;
                const uint32_t k = d.kf[r.aln];
                if (k != 0 && e_end > P0 && r.gstart < P0 + (uint32_t)TL_T) d.wrec[i] = make_uint4(r.aln, r.gstart, general_walk<BITS>(S, r, k, PoolBases<BITS>(d, r)), k);
            }
        }
        __syncwarp();          // lanes that had a queued read rejoin their warp here: without it the warp may run phase C in two groups
        __syncthreads();
#ifdef PP_TILE_PROF
        pt[3] = clock64();
#endif
        // ---- phase C: difference arrays -> cover per position, and the deficit where alignments with k != 1 touch the tile.  After
        // the scans every thread only reads and writes its own positions of `deficit` / `depth`: no barrier until the end of the tile.
        const uint32_t rel0 = tid * TL_PER_THREAD;
        uint32_t cover[TL_PER_THREAD];
        uint32_t multi = 0;                                  // bit i: position rel0 + i has k != 1 coverage (depth from the deficit)
        {
            long long csum = 0;
#pragma unroll
            for (int i = 0; i < TL_PER_THREAD; ++i) { csum += sh.cdiff[rel0 + i]; cover[i] = (uint32_t)csum; }
            const unsigned long long ex = block_exscan<TL_THREADS>((unsigned long long)csum, sh.s_warp, &sh.s_total);
#pragma unroll
            for (int i = 0; i < TL_PER_THREAD; ++i) cover[i] += (uint32_t)ex;
            if (sh.any_multi) {                              // (block-uniform)
                unsigned long long dsum = 0, dv[TL_PER_THREAD];
#pragma unroll
                for (int i = 0; i < TL_PER_THREAD; ++i) { dsum += sh.deficit[rel0 + i]; dv[i] = dsum; }
                const unsigned long long dex = block_exscan<TL_THREADS>(dsum, sh.s_warp, &sh.s_total);
#pragma unroll
                for (int i = 0; i < TL_PER_THREAD; ++i) {
                    sh.deficit[rel0 + i] = dv[i] + dex;
                    if (dv[i] + dex != 0 || cover[i] >= TL_DEF_COVER) multi |= 1u << i;
                }
            }
        }
#ifdef PP_TILE_PROF
        pt[4] = clock64();
#endif
        // ---- phase D: the ordered depth walk, where the deficit's bound cannot settle the vote.  Warp w owns sub-tile w here AND in
        // the vote below.  A position decides the vote without depth when no allele other than the draft's can reach the valid
        // threshold (the same tests as in phase E, on the lower bound), else when both ends of the bound give the same thresholds.
        // The debug records print depth itself: there every sub-tile with k != 1 coverage walks.  The change records print it too:
        // there a sub-tile also walks when one of its positions passes these tests, which every position that reaches the vote does.
        bool walk;
        {
            bool open = false;
            if (multi && !vp.dbg) {
#pragma unroll
                for (int i = 0; i < TL_PER_THREAD; ++i) {
                    if (!((multi >> i) & 1u)) continue;
                    const uint32_t rel = rel0 + i;
                    if (cover[i] >= TL_DEF_COVER) { open = true; continue; }
                    const uint32_t mx = max(max(max(sh.ex[0][rel], sh.ex[1][rel]), max(sh.ex[2][rel], sh.ex[3][rel])), max(sh.del[rel], sh.oth[rel]));
                    if (mx == 0 || mx < prm.min_depth) continue;
                    const DepthBounds db = depth_bounds(cover[i], sh.deficit[rel]);
                    if ((double)mx + 2.0 < db.lo * prm.fv) continue;
                    if (CHG || !same_thresholds(prm, db.lo, db.hi)) open = true;
                }
            }
            walk = __ballot_sync(0xffffffffu, vp.dbg ? multi != 0 : open) != 0;
        }
#ifdef PP_TILE_PROF
        const long long dw0 = clock64();
#endif
        if (walk) depth_walk<BITS>(d, sh, sh.wstage[warp], P0, warp, lb, long_lo, long_hi);
#ifdef PP_TILE_PROF
        if (lane == 0 && walk) { atomicAdd(&d.st->prof[8], (unsigned long long)(clock64() - dw0)); atomicAdd(&d.st->prof[9], 1ull); }
#endif
        __syncwarp();
        // ---- phase E: the vote, straight out of shared memory
        const uint32_t p0 = P0 + rel0;
        PosOut po[TL_PER_THREAD];
        unsigned long long tlen = 0;
        uint32_t n_changed = 0, n_zero = 0;
        double tdepth = 0.0;
        uint32_t ctg = 0;
        if (p0 < d.G) {
            uint32_t clo = 0, chi = d.n_contigs;           // largest c with contig_off[c] <= p0
            while (chi - clo > 1) { const uint32_t mid = (clo + chi) >> 1; if (d.contig_off[mid] <= p0) clo = mid; else chi = mid; }
            ctg = clo;
        }
        uint32_t next_start = (ctg + 1 < d.n_contigs) ? (uint32_t)d.contig_off[ctg + 1] : 0xFFFFFFFFu;
        const uint32_t dr = *reinterpret_cast<const uint32_t*>(d.draft + p0);      // draft is padded past G
#pragma unroll
        for (int i = 0; i < TL_PER_THREAD; ++i) {
            const uint32_t p = p0 + i;
            po[i].packed = 0; po[i].rec = 0;
            if (p >= d.G) continue;
            while (p >= next_start) {
                if (n_changed) atomicAdd(&vp.changed[ctg], (unsigned long long)n_changed);
                if (n_zero) atomicAdd(&vp.zero_depth[ctg], (unsigned long long)n_zero);
                if (tdepth != 0.0) atomicAdd(&vp.total_depth[ctg], tdepth);
                n_changed = n_zero = 0;
                tdepth = 0.0;
                ctg++;
                next_start = (ctg + 1 < d.n_contigs) ? (uint32_t)d.contig_off[ctg + 1] : 0xFFFFFFFFu;
            }
            const uint32_t orig = (dr >> (i * 8)) & 255u;
            const uint32_t cov = cover[i];
            if (cov == 0) {                                    // depth 0: always the original base
                n_zero++;
                po[i].packed = (orig == '-' ? 0u : 1u) | (orig << 16);
                tlen += po[i].packed & 0xFFFFu;
                if (vp.dbg) {                                  // min_depth > 0: low_depth; min_depth == 0: A,C,G,T all "valid" -> multiple
                    pp_debug_pos r;
                    memset(&r, 0, sizeof r);
                    r.valid_threshold = prm.min_depth; r.new_node = 0xFFFFFFFFu; r.original = (uint8_t)orig;
                    r.status = prm.min_depth > 0 ? 0 : 2; r.new_char = (uint8_t)orig;
                    vp.dbg[p] = r;
                }
                continue;
            }
            const uint32_t rel = rel0 + i;
            // depth: the reference's where it is known (no k != 1 coverage, or the warp walked), else the fixed-point estimate
            // (per-contig statistics only).  vdepth, what the vote reads: there the lower bound, whose thresholds phase D found
            // to be the reference's.
            double depth = (double)cov, vdepth = depth;
            if ((multi >> i) & 1u) {
                if (walk) depth = vdepth = sh.depth[rel];
                else { const DepthBounds db = depth_bounds(cov, sh.deficit[rel]); depth = db.fx; vdepth = db.lo; }
            }
            tdepth += depth;
            uint32_t cA = sh.ex[0][rel], cC = sh.ex[1][rel], cG = sh.ex[2][rel], cT = sh.ex[3][rel];
            const uint32_t cDel = sh.del[rel], n_other = sh.oth[rel];
            if ((cA | cC | cG | cT | cDel | n_other) == 0 && !vp.dbg) {
                // every covering entry equals the draft base: the only allele with a non-zero count is the draft's own, so
                // whatever the thresholds say (kept, too_close, low_depth, ...) the emitted base is the original
                po[i].packed = (orig == '-' ? 0u : 1u) | (orig << 16);
                tlen += po[i].packed & 0xFFFFu;
                continue;
            }
            if (!vp.dbg) {
                // The emitted base differs from the draft only if an allele OTHER than the draft's reaches the valid threshold
                // max(min_depth, round(depth * fraction_valid)) (pileup.rs:70-72,114-129).  No such allele can when the largest
                // non-draft count is below min_depth, or below depth * fraction_valid by more than rounding can bridge: the
                // position keeps its base whatever its status (kept / too_close / low_depth / none / multiple).
                const uint32_t mx = max(max(max(cA, cC), max(cG, cT)), max(cDel, n_other));
                if (mx < prm.min_depth || (double)mx + 2.0 < vdepth * prm.fv) {
                    po[i].packed = (orig == '-' ? 0u : 1u) | (orig << 16);
                    tlen += po[i].packed & 0xFFFFu;
                    continue;
                }
            }
            uint32_t matched = cov - (cA + cC + cG + cT + cDel + n_other);
            if (orig == 'A') { cA += matched; matched = 0; }
            else if (orig == 'C') { cC += matched; matched = 0; }
            else if (orig == 'G') { cG += matched; matched = 0; }
            else if (orig == 'T') { cT += matched; matched = 0; }
            po[i] = vote_position<BITS, CHG>(oc, prm, p, orig, vdepth, cA, cC, cG, cT, cDel, matched, n_other, vp);
            n_changed += (po[i].packed >> 24) & 1u;
            tlen += po[i].packed & 0xFFFFu;
        }
        {   // per-contig statistics: one atomic per warp when the whole warp sits in one contig (nearly always)
            const uint32_t ctg0 = __shfl_sync(0xffffffffu, ctg, 0);
            if (__ballot_sync(0xffffffffu, ctg != ctg0) == 0u) {
                for (int o = 16; o > 0; o >>= 1) {
                    n_changed += __shfl_down_sync(0xffffffffu, n_changed, o);
                    n_zero += __shfl_down_sync(0xffffffffu, n_zero, o);
                    tdepth += __shfl_down_sync(0xffffffffu, tdepth, o);
                }
                if (lane != 0) { n_changed = n_zero = 0; tdepth = 0.0; }
            }
            if (n_changed) atomicAdd(&vp.changed[ctg], (unsigned long long)n_changed);
            if (n_zero) atomicAdd(&vp.zero_depth[ctg], (unsigned long long)n_zero);
            if (tdepth != 0.0) atomicAdd(&vp.total_depth[ctg], tdepth);
        }
        // hand the verdicts to k_compact: 2 bytes per position + this tile's length delta
        {
            uint32_t w2[TL_PER_THREAD / 2];
#pragma unroll
            for (int i = 0; i < TL_PER_THREAD; ++i) {
                const uint32_t len = po[i].packed & 0xFFFFu;
                uint32_t h;
                if ((po[i].packed >> 25) & 1u) { h = 255u << 8; if (p0 + i < d.G) vp.rec_at[p0 + i] = po[i].rec; }
                else h = (len << 8) | ((po[i].packed >> 16) & 255u);
                if (i & 1) w2[i >> 1] |= h << 16; else w2[i >> 1] = h;
            }
            *reinterpret_cast<uint2*>(vp.res + p0) = make_uint2(w2[0], w2[1]);
        }
        const uint32_t npos = (p0 < d.G) ? min((uint32_t)TL_PER_THREAD, d.G - p0) : 0u;
        long long delta = (long long)tlen - (long long)npos;
        for (int o = 16; o > 0; o >>= 1) delta += __shfl_down_sync(0xffffffffu, delta, o);
        if (lane == 0) sh.s_delta[warp] = delta;
#ifdef PP_TILE_PROF
        if (__syncthreads_or(walk) && tid == 0) atomicAdd(&d.st->prof[10], 1ull);
#endif
        __syncthreads();
        if (tid == 0) {
            long long t = 0;
            for (int i = 0; i < TL_THREADS / 32; ++i) t += sh.s_delta[i];
            vp.chunk_delta[tile] = t;
#ifdef PP_TILE_PROF
            pt[5] = clock64();
            for (int i = 0; i < 5; ++i) atomicAdd(&d.st->prof[i], (unsigned long long)(pt[i + 1] - pt[i]));
            atomicAdd(&d.st->prof[5], (unsigned long long)sh.qn);
            atomicAdd(&d.st->prof[6], 1ull);
            atomicMax(&d.st->prof[7], (unsigned long long)sh.qn);
#endif
        }
    }
}
static_assert(TL_PER_THREAD == 4, "the verdict store packs four positions per thread");

#if !defined(PP_EMULATE)
// One CTA per SM: built for sm_90a, the body needs ~100 registers per thread.  Capped at 64 for two CTAs per SM it spills, and on an
// H100 (400 W) the tile kernel took 0.79 ms per 5 Mbp x 100x call that way against 0.71 ms with one CTA per SM.
template <int BITS, bool CHG>
__global__ void __launch_bounds__(TL_THREADS, 1) k_tile(DevData d, VoteParams vp) {
    extern __shared__ __align__(16) unsigned char tile_smem[];
    tile_body<BITS, CHG>(d, vp, *reinterpret_cast<TileShared*>(tile_smem));
}
#endif

// ------------------------------------------------------------------------------------------------------
// k_allele_strings: the strings behind debug and change records (the keys of the reference's HashMap<String,u32>, pileup.rs:62),
// so that a report never needs the alignments on the host.  Runs after a polish call, on its chains.  Row i (global position
// pos[i], record rec[by_pos ? pos[i] : i]) gets, at pool + off[i]: u32 n, then n times (u32 count, u32 length, the characters)
// for the position's other alleles in chain order, then u32 length and the characters of the emitted allele when that is a node
// (length 0 otherwise); little-endian.  Space is taken with one atomicAdd per row on *used: where *used ends above cap, rows were
// left unwritten and the call is repeated with a pool of *used bytes.
// ------------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint8_t* put_u32(uint8_t* w, uint32_t v) {
    w[0] = (uint8_t)v; w[1] = (uint8_t)(v >> 8); w[2] = (uint8_t)(v >> 16); w[3] = (uint8_t)(v >> 24);
    return w + 4;
}
template <int BITS>
__device__ void allele_strings_row(const OthCtx& oc, uint32_t pos, uint32_t new_node, uint8_t* pool, unsigned long long cap,
                                   unsigned long long* used, unsigned long long* off) {
    unsigned long long bytes = 8;
    uint32_t n = 0;
    for (uint32_t nd = oc.head[pos]; nd != 0; nd = oc.nodes[nd - 1].next == NONE32 ? 0 : oc.nodes[nd - 1].next + 1) {
        bytes += 8 + ((uint32_t)oc.nodes[nd - 1].val & 0xFFFFu);
        n++;
    }
    const uint32_t new_len = new_node == NONE32 ? 0u : (uint32_t)oc.nodes[new_node].val & 0xFFFFu;
    bytes += new_len;
    const unsigned long long o = atomicAdd(used, bytes);
    *off = o;
    if (o + bytes > cap) return;
    uint8_t* w = put_u32(pool + o, n);
    for (uint32_t nd = oc.head[pos]; nd != 0; nd = oc.nodes[nd - 1].next == NONE32 ? 0 : oc.nodes[nd - 1].next + 1) {
        const uint32_t len = (uint32_t)oc.nodes[nd - 1].val & 0xFFFFu;
        w = put_u32(put_u32(w, oc.nodes[nd - 1].count), len);
        for (uint32_t t = 0; t < len; ++t) *w++ = other_char<BITS>(oc, nd - 1, t);
    }
    w = put_u32(w, new_len);
    for (uint32_t t = 0; t < new_len; ++t) *w++ = other_char<BITS>(oc, new_node, t);
}
template <int BITS>
__device__ void allele_strings_body(const OthCtx& oc, const uint32_t* pos, const pp_debug_pos* rec, bool by_pos, uint32_t n, uint8_t* pool,
                                    unsigned long long cap, unsigned long long* used, unsigned long long* off) {
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const uint32_t p = pos[i];
        allele_strings_row<BITS>(oc, p, rec[by_pos ? p : i].new_node, pool, cap, used, off + i);
    }
}
#if !defined(PP_EMULATE)
template <int BITS>
__global__ void __launch_bounds__(256) k_allele_strings(OthCtx oc, const uint32_t* pos, const pp_debug_pos* rec, bool by_pos, uint32_t n,
                                                         uint8_t* pool, unsigned long long cap, unsigned long long* used, unsigned long long* off) {
    allele_strings_body<BITS>(oc, pos, rec, by_pos, n, pool, cap, used, off);
}
#endif

// ------------------------------------------------------------------------------------------------------
// k_compact: polish.rs:185-188 (push_str of every position's allele, then replace("-", "")).  Chunk c writes its
// characters at c * VT_CHUNK + sum(chunk_delta[0..c)); no inter-CTA dependency.
// ------------------------------------------------------------------------------------------------------
#define CP_STAGE (VT_CHUNK + 2048)
struct CompactShared {
    unsigned long long s_warp[VT_THREADS / 32];
    unsigned long long s_total;
    long long s_red[VT_THREADS / 32];
    long long s_base;
    __align__(16) uint8_t s_out[CP_STAGE];
};

template <int BITS>
__device__ __forceinline__ void compact_body(const DevData& d, const VoteParams& vp, CompactShared& sh) {
    const uint32_t tid = threadIdx.x, chunk = blockIdx.x;
    const uint32_t p0 = chunk * VT_CHUNK + tid * VT_ITEMS;
    // base offset of this chunk
    long long acc = 0;
    for (uint32_t j = tid; j < chunk; j += VT_THREADS) acc += vp.chunk_delta[j];
    for (int o = 16; o > 0; o >>= 1) acc += __shfl_down_sync(0xffffffffu, acc, o);
    if ((tid & 31) == 0) sh.s_red[tid >> 5] = acc;
    __syncthreads();
    if (tid == 0) {
        long long t = 0;
        for (int i = 0; i < VT_THREADS / 32; ++i) t += sh.s_red[i];
        sh.s_base = (long long)chunk * VT_CHUNK + t;
    }
    // verdicts
    const uint4 rv = *reinterpret_cast<const uint4*>(vp.res + p0);
    const uint32_t w[4] = {rv.x, rv.y, rv.z, rv.w};
    uint32_t len[VT_ITEMS];
    unsigned long long tlen = 0;
    OthCtx oc;
    oc.nodes = d.nodes; oc.head = d.oth_head;
    oc.sr = SeqRef{d.seq_pool, d.seq_off, d.seq_len, d.flags};
#pragma unroll
    for (int i = 0; i < VT_ITEMS; ++i) {
        const uint32_t h = (w[i >> 1] >> ((i & 1) * 16)) & 0xFFFFu;
        uint32_t l = h >> 8;
        if (p0 + i >= d.G) l = 0;
        else if (l == 255) {                                      // a multi-base allele: count its non-'-' characters
            const uint32_t rec = vp.rec_at[p0 + i];
            const uint32_t rlen = (uint32_t)oc.nodes[rec].val & 0xFFFFu;
            l = 0;
            for (uint32_t t = 0; t < rlen; ++t) l += other_char<BITS>(oc, rec, t) != '-';
        }
        len[i] = l;
        tlen += l;
    }
    const unsigned long long oexcl = block_exscan<VT_THREADS>(tlen, sh.s_warp, &sh.s_total);
    const unsigned long long total = sh.s_total;
    const unsigned long long base = (unsigned long long)sh.s_base;
    if (chunk == vp.n_chunks - 1 && tid == 0) { vp.out_off[d.n_contigs] = base + total; d.st->out_len = base + total; }
    // out_off of contigs that start inside this thread's positions
    if (p0 < d.G) {
        uint32_t lo = 0, hi = d.n_contigs;           // first c with contig_off[c] >= p0
        while (lo < hi) { const uint32_t mid = (lo + hi) >> 1; if (d.contig_off[mid] < p0) lo = mid + 1; else hi = mid; }
        if (lo < d.n_contigs && d.contig_off[lo] < (unsigned long long)p0 + VT_ITEMS) {
            unsigned long long oo = base + oexcl;
            uint32_t c = lo;
#pragma unroll
            for (int i = 0; i < VT_ITEMS; ++i) {
                while (c < d.n_contigs && d.contig_off[c] == p0 + i) { vp.out_off[c] = oo; c++; }
                oo += len[i];
            }
        }
    }
    if (base + total > vp.out_cap) { if (tid == 0) atomicOr(&d.st->flags, (unsigned)FL_OUT_OVF); return; }
    const bool staged = total <= CP_STAGE;
    uint8_t* dst = staged ? sh.s_out : vp.out + base;
    unsigned long long o = oexcl;
#pragma unroll
    for (int i = 0; i < VT_ITEMS; ++i) {
        if (len[i] == 0) continue;
        const uint32_t h = (w[i >> 1] >> ((i & 1) * 16)) & 0xFFFFu;
        if ((h >> 8) != 255) { dst[o++] = (uint8_t)h; continue; }
        const uint32_t rec = vp.rec_at[p0 + i];
        const uint32_t rlen = (uint32_t)oc.nodes[rec].val & 0xFFFFu;
        for (uint32_t t = 0; t < rlen; ++t) {
            const uint8_t ch = other_char<BITS>(oc, rec, t);
            if (ch != '-') dst[o++] = ch;                          // polish.rs:188 replace("-", "")
        }
    }
    if (!staged) return;
    __syncthreads();
    // coalesced copy of the staged bytes: head to a 16-byte boundary, body as uint4, tail
    uint8_t* g = vp.out + base;
    const uint32_t n = (uint32_t)total;
    const uint32_t head = min(n, (uint32_t)((16 - ((size_t)g & 15)) & 15));
    for (uint32_t i = tid; i < head; i += VT_THREADS) g[i] = sh.s_out[i];
    const uint32_t nvec = (n - head) / 16;
    for (uint32_t i = tid; i < nvec; i += VT_THREADS) {
        const uint8_t* sp = sh.s_out + head + i * 16;
        uint32_t x[4];
#pragma unroll
        for (int k = 0; k < 4; ++k) x[k] = sp[4 * k] | (sp[4 * k + 1] << 8) | (sp[4 * k + 2] << 16) | ((uint32_t)sp[4 * k + 3] << 24);
        reinterpret_cast<uint4*>(g + head)[i] = make_uint4(x[0], x[1], x[2], x[3]);
    }
    for (uint32_t i = head + nvec * 16 + tid; i < n; i += VT_THREADS) g[i] = sh.s_out[i];
}

#if !defined(PP_EMULATE)
template <int BITS>
__global__ void __launch_bounds__(VT_THREADS) k_compact(DevData d, VoteParams vp) {
    __shared__ CompactShared sh;
    compact_body<BITS>(d, vp, sh);
}
#endif
