// emu_depth.cpp — the polish kernels of polypolish_b200/csrc/polish_dev.cuh on the CPU (tests/emu/cuda_emu.h) with the per-position
// reports recorded: k_tile<BITS, CHG, STS, true>'s depth keys (and, STS, its status bytes after them, as in the product's one buffer),
// then k_status_heads<T>, the exclusive scan of its counts (CUB's on the device, std::exclusive_scan here) and k_status_runs<T> for
// each report, then the runs as the lines `polish --depth-bedgraph` / `polish --status-bed` write.  The launch sequence is
// emu_status.cpp's.  Also depth_tenths and the host's depth text against snprintf("%.1f").
// TEST INFRASTRUCTURE: built and used by tests/test_emu_depth.py only; nothing in polypolish_b200/ links or loads this.
#include "cuda_emu.h"

#include "../../polypolish_b200/csrc/polish_dev.cuh"
#include "../../polypolish_b200/csrc/debug_rows.h"

#include <numeric>
#include <string>

namespace {

void init_comp_table() {
    for (int i = 0; i < 256; ++i) c_comp[i] = 'N';
    const char* a = "ATGCNRYSWKMBVDH.-?";
    const char* b = "TACGNYRSWMKVBHD.-?";
    for (int i = 0; a[i]; ++i) c_comp[(unsigned char)a[i]] = (uint8_t)b[i];
}

// The runs of one report as "<contig>\t<start>\t<end>\t<value>" lines; 101: the runs are malformed (an empty run or one that
// crosses a contig).
template <class T, class Text>
int runs_text(const pp_contigs* c, const T* e, const char* const* names, Text text, std::string* out) {
    const uint64_t G = c->off[c->n_contigs];
    const uint32_t n_blk = (uint32_t)((G + SR_CHUNK - 1) / SR_CHUNK);
    std::vector<uint32_t> first(n_blk + 1, 0);
    emu::launch(n_blk, SR_THREADS, sizeof(RunShared), [&] { status_heads_body(e, (uint32_t)G, first.data(), *(RunShared*)emu::shared_base()); });
    std::exclusive_scan(first.begin(), first.end(), first.begin(), 0u);
    const uint32_t n = first[n_blk];
    std::vector<uint32_t> start(n + 1, 0xEEEEEEEEu);
    std::vector<T> value(n + 1, (T)0xEE);
    emu::launch(n_blk, SR_THREADS, sizeof(RunShared), [&] {
        status_runs_body(e, (uint32_t)G, first.data(), start.data(), value.data(), *(RunShared*)emu::shared_base());
    });
    for (uint32_t i = 0; i < n; ++i) {
        const uint32_t ctg = (uint32_t)(std::upper_bound(c->off, c->off + c->n_contigs + 1, (uint64_t)start[i]) - c->off) - 1;
        const uint64_t end = i + 1 < n ? start[i + 1] : G;
        if (end <= start[i] || end > c->off[ctg + 1]) return 101;
        *out += std::string(names[ctg]) + "\t" + std::to_string(start[i] - c->off[ctg]) + "\t" + std::to_string(end - c->off[ctg]) + "\t";
        text(*out, value[i]);
        *out += "\n";
    }
    return 0;
}

template <int BITS, bool CHG, bool STS>
int run(const pp_contigs* c, const pp_alignments* a, const pp_polish_params* prm, pp_polish_result* res, int grid_tiles, bool global_k,
        uint64_t* err_out, const char* const* names, std::string* bed, std::string* bedgraph) {
    const uint64_t G = c->off[c->n_contigs], n_aln = a->n_aln;
    const uint32_t n_tiles = (uint32_t)((G + TL_T - 1) / TL_T), n_bins = (uint32_t)((G + PP_BIN - 1) >> PP_BIN_SHIFT);
    const size_t padG = (size_t)n_tiles * TL_T + 16;
    std::vector<uint8_t> draft(padG + 4096, 0);
    memcpy(draft.data(), c->bases, G);
    std::vector<uint8_t> seq_pool(a->seq_pool_bytes + 512, 0);
    if (a->seq_pool_bytes) memcpy(seq_pool.data(), a->seq_pool, a->seq_pool_bytes);
    // 16-byte aligned copies (uint4 loads)
    std::vector<uint4> draft16((draft.size() + 15) / 16), pool16((seq_pool.size() + 15) / 16);
    memcpy(draft16.data(), draft.data(), draft.size());
    memcpy(pool16.data(), seq_pool.data(), seq_pool.size());
    std::vector<uint32_t> cigar_ops(a->n_cigar_ops + 16, 0);
    if (a->n_cigar_ops) memcpy(cigar_ops.data(), a->cigar_ops, a->n_cigar_ops * 4);

    std::vector<TileRec> recs(n_aln + 16), srec(n_aln + 16);
    std::vector<uint32_t> key(n_aln + 16), val(n_aln + 16), skey(n_aln + 16), sval(n_aln + 16), bin_start(n_bins + 4, 0), kf(n_aln + 16, 0xDEADBEEFu);
    std::vector<uint4> wrec(n_aln + 16, make_uint4(0xDEADBEEFu, 0xDEADBEEFu, 0xDEADBEEFu, 0xDEADBEEFu));
    std::vector<uint4> sseq((n_aln + 16) * TL_SEQ_QUADS + 16, make_uint4(0xCDCDCDCDu, 0xCDCDCDCDu, 0xCDCDCDCDu, 0xCDCDCDCDu));
    std::vector<uint8_t> errc(n_aln + 16, 0xEE);
    std::vector<uint16_t> gq(n_aln + 16, 0xEEEE);
    std::vector<uint32_t> oth_head(((size_t)(G + TL_T - 1) / TL_T) * TL_T + 16, 0xEEEEEEEEu), kcount(a->n_reads + 2, 0);   // (k_tile zeroes the heads itself)
    std::vector<OthNode> nodes(std::max<uint64_t>(1 << 16, n_aln * 4 + G));
    std::vector<unsigned long long> changed(c->n_contigs, 0), zero(c->n_contigs, 0), out_off(c->n_contigs + 1, 0);
    std::vector<double> tdepth(c->n_contigs, 0.0);
    std::vector<uint16_t> resv(padG, 0);
    std::vector<uint32_t> rec_at(G + 1, 0);
    std::vector<long long> chunk_delta(n_tiles, 0);
    const uint64_t out_cap = G + G / 4 + (1u << 20);
    std::vector<uint8_t> out(out_cap + 64);
    DevStatus st;
    memset(&st, 0, sizeof st);
    st.err = ~0ull;
    DevParams dp{prm->fraction_valid, prm->fraction_invalid, prm->min_depth, prm->max_errors, prm->careful ? 1 : 0, 0};

    DevData d;
    memset(&d, 0, sizeof d);
    d.n_aln = n_aln;
    d.contig = a->contig; d.ref_start = a->ref_start; d.read_id = a->read_id; d.seq_off = a->seq_off; d.cigar_off = a->cigar_off; d.nm = a->nm;
    d.cigar_ops = cigar_ops.data(); d.seq_len = a->seq_len; d.n_cigar = a->n_cigar; d.flags = a->flags;
    d.seq_pool = (const uint8_t*)pool16.data(); d.draft = (const uint8_t*)draft16.data();
    d.contig_off = (const unsigned long long*)c->off; d.n_contigs = c->n_contigs; d.G = (uint32_t)G; d.n_bins = n_bins; d.n_tiles = n_tiles;
    d.k = kcount.data(); d.recs = recs.data(); d.key = key.data(); d.val = val.data(); d.sval = sval.data(); d.bin_start = bin_start.data();
    d.srec = srec.data(); d.sseq = sseq.data(); d.kf = kf.data(); d.errc = errc.data(); d.gq = gq.data();
    d.wrec = wrec.data(); d.oth_head = oth_head.data(); d.nodes = nodes.data(); d.node_cap = (uint32_t)nodes.size(); d.prm = &dp; d.st = &st;
    VoteParams vp;
    vp.n_chunks = n_tiles; vp.out = out.data(); vp.out_cap = out_cap; vp.out_off = out_off.data(); vp.changed = changed.data();
    vp.zero_depth = zero.data(); vp.total_depth = tdepth.data(); vp.res = resv.data(); vp.rec_at = rec_at.data(); vp.chunk_delta = chunk_delta.data();
    vp.dbg = nullptr;
    // the change list (CHG), with room for every position: it never overflows here
    std::vector<pp_debug_pos> chg(G + 1);
    std::vector<uint32_t> chg_pos(G + 1);
    vp.chg = chg.data(); vp.chg_pos = chg_pos.data(); vp.chg_n = &st.n_changes; vp.chg_cap = (uint32_t)chg.size();
    // the depth keys, then the status bytes, padded like the product's (run_polish in polish_kernels.cu); the padding is never read
    const uint32_t n_blk = (uint32_t)((G + SR_CHUNK - 1) / SR_CHUNK);
    const size_t key_bytes = depth_key_bytes(G);
    std::vector<uint4> rep16((key_bytes + (size_t)n_blk * SR_CHUNK) / 16 + 1, make_uint4(0xA5A5A5A5u, 0xA5A5A5A5u, 0xA5A5A5A5u, 0xA5A5A5A5u));
    vp.sts = (uint8_t*)rep16.data();

    // ---- once per dataset: bin, stable sort, bounds, permute
    if (n_aln) {
        emu::launch(3, 256, 0, [&] { bin_body<BITS>(d); });
        std::vector<uint32_t> order(n_aln);
        std::iota(order.begin(), order.end(), 0u);
        std::stable_sort(order.begin(), order.end(), [&](uint32_t x, uint32_t y) { return key[x] < key[y]; });   // = the stable radix sort
        for (uint64_t i = 0; i < n_aln; ++i) { skey[i] = key[order[i]]; sval[i] = val[order[i]]; }
    }
    emu::launch((unsigned)((n_aln + 1 + 255) / 256), 256, 0, [&] { bin_bounds_body(skey.data(), (uint32_t)n_aln, n_bins + 2, bin_start.data()); });
    d.n_slots = bin_start[n_bins + 1];
    d.max_ext = st.max_ext;
    if (st.flags & FL_PAST_END) emu::launch(2, 256, 0, [&] { past_end_body<BITS>(d); });   // (after the pool is there, as on the device)
    if (d.n_slots) {
        emu::launch((d.n_slots + 255) / 256, 256, 0, [&] { permute_body(d); });
        if (BITS == 4) emu::launch((unsigned)(((uint64_t)d.n_slots * TL_SEQ_QUADS + 255) / 256), 256, 0, [&] { permute_seq_body(d); });
    }
    std::vector<uint32_t> tweight(n_tiles + 1), tindex(n_tiles + 1), torder(n_tiles + 1);
    emu::launch((n_tiles + 255) / 256, 256, 0, [&] { tile_weight_body(d, tweight.data(), tindex.data()); });
    {
        std::vector<uint32_t> o(n_tiles);
        std::iota(o.begin(), o.end(), 0u);
        std::stable_sort(o.begin(), o.end(), [&](uint32_t x, uint32_t y) { return tweight[x] > tweight[y]; });
        for (uint32_t i = 0; i < n_tiles; ++i) torder[i] = tindex[o[i]];
    }
    d.tile_order = torder.data();
    // ---- per call
    if (n_aln && global_k) emu::launch(2, 256, 0, [&] { k_classify_multi(d); });
    if (n_aln)
        emu::launch(2, PR_THREADS, sizeof(PrepShared), [&] {
            PrepShared& sh = *(PrepShared*)emu::shared_base();
            if (global_k) goodk_body<true>(d, sh); else goodk_body<false>(d, sh);
        });
    emu::launch((unsigned)std::max(1, std::min<int>(grid_tiles, (int)n_tiles)), TL_THREADS, sizeof(TileShared), [&] {
        tile_body<BITS, CHG, STS, true>(d, vp, *(TileShared*)emu::shared_base());
    });
    emu::launch(n_tiles, VT_THREADS, sizeof(CompactShared), [&] { compact_body<BITS>(d, vp, *(CompactShared*)emu::shared_base()); });

    if (st.err == ~0ull) {                                  // the runs, then the lines contig by contig
        const int rc = runs_text(c, (const unsigned long long*)vp.sts, names, [](std::string& o, unsigned long long t) { pp::depth_text(o, t); }, bedgraph);
        if (rc) return rc;
        if (STS) {
            static const char* const word[6] = {"low_depth", "none", "multiple", "too_close", "kept", "changed"};
            const int rs = runs_text(c, vp.sts + key_bytes, names, [](std::string& o, uint8_t s) { o += s < 6 ? word[s] : "?"; }, bed);
            if (rs) return rs;
        }
    }
    *err_out = st.err;
    res->out_len = st.out_len;
    res->n_aln_used = st.n_used;
    res->error_aln = st.err == ~0ull ? -1 : (int64_t)(st.err >> 8);
    if (st.err != ~0ull) return PP_ERR_INPUT;
    if (st.flags & FL_BIGGROUP) return 100;
    if (st.flags & (FL_NODE_OVF | FL_OUT_OVF)) return PP_ERR_NOMEM;
    if (res->out_bases) {
        if (res->out_cap < st.out_len) return PP_ERR_ARG;
        memcpy(res->out_bases, out.data(), st.out_len);
        if (res->out_off) memcpy(res->out_off, out_off.data(), (c->n_contigs + 1) * 8);
        if (res->changed) memcpy(res->changed, changed.data(), c->n_contigs * 8);
        if (res->zero_depth) memcpy(res->zero_depth, zero.data(), c->n_contigs * 8);
        if (res->total_depth) memcpy(res->total_depth, tdepth.data(), c->n_contigs * 8);
    }
    return PP_OK;
}

template <int BITS>
int run_any(bool chg, bool sts, const pp_contigs* c, const pp_alignments* a, const pp_polish_params* prm, pp_polish_result* res, int grid_tiles,
            bool global_k, uint64_t* err, const char* const* names, std::string* bed, std::string* bedgraph) {
    if (chg) return sts ? run<BITS, true, true>(c, a, prm, res, grid_tiles, global_k, err, names, bed, bedgraph)
                        : run<BITS, true, false>(c, a, prm, res, grid_tiles, global_k, err, names, bed, bedgraph);
    return sts ? run<BITS, false, true>(c, a, prm, res, grid_tiles, global_k, err, names, bed, bedgraph)
               : run<BITS, false, false>(c, a, prm, res, grid_tiles, global_k, err, names, bed, bedgraph);
}

}  // namespace

// The polish kernels on the CPU in depth mode: names = the contigs' names; *bedgraph (free with emu_free) receives the bytes
// `polish --depth-bedgraph` writes, and with with_status *bed those of `polish --status-bed` from the same call.  with_changes: the
// change report is recorded in the same call.  grid_tiles = CTAs of k_tile.  101: the runs are malformed.
extern "C" int emu_polish_depth(const pp_contigs* c, const pp_alignments* a, const pp_polish_params* prm, pp_polish_result* res, int grid_tiles,
                                int with_changes, int with_status, unsigned long long* err_code, const char* const* names, char** bedgraph,
                                char** bed) {
    init_comp_table();
    uint64_t err = 0;
    std::string out, out_bed;
    auto go = [&](bool global_k) {
        out.clear(); out_bed.clear();
        return a->seq_bits == 4 ? run_any<4>(with_changes, with_status, c, a, prm, res, grid_tiles, global_k, &err, names, &out_bed, &out)
                                : run_any<8>(with_changes, with_status, c, a, prm, res, grid_tiles, global_k, &err, names, &out_bed, &out);
    };
    int rc = go(false);
    if (rc == 100) rc = go(true);
    if (err_code) *err_code = err;
    *bedgraph = strdup(out.c_str());
    *bed = strdup(out_bed.c_str());
    return rc;
}

// depth_tenths(x[i]) into tenths[i]; returns the first i whose depth text (pp::depth_text of the tenths) is not snprintf("%.1f", x[i]),
// or n when there is none.
extern "C" uint64_t emu_depth_tenths(const double* x, uint64_t n, unsigned long long* tenths) {
    std::string t;
    char want[512];
    for (uint64_t i = 0; i < n; ++i) {
        tenths[i] = depth_tenths(x[i]);
        t.clear();
        pp::depth_text(t, tenths[i]);
        snprintf(want, sizeof want, "%.1f", x[i]);
        if (t != want) return i;
    }
    return n;
}

// pp::depth_text of each key, one per line (free with emu_free)
extern "C" char* emu_depth_text(const unsigned long long* tenths, uint64_t n) {
    std::string t;
    for (uint64_t i = 0; i < n; ++i) { pp::depth_text(t, tenths[i]); t += '\n'; }
    return strdup(t.c_str());
}

extern "C" void emu_free(void* p) { free(p); }
