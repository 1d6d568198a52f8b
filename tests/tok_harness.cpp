// CPU harness for the device SAM tokeniser's per-item logic (polypolish_b200/csrc/tok_line.h, tok_table.h): runs the
// kernels' bodies item by item in the order of the device pipeline (line index -> parse -> scans -> emit -> group heads ->
// read ids -> group close), so that tests/test_tok_cpu.py can compare the arrays with the host packer's without a GPU.
// Compiled by the test with g++.
#include <algorithm>
#include <cstdint>
#include <cstring>
#include <string>
#include <vector>

#include "../polypolish_b200/csrc/tok_line.h"
#include "../polypolish_b200/csrc/tok_table.h"

extern "C" int tok_cpu(const char* text_in, uint64_t n, const char* const* names, uint32_t n_names, int careful, int bits,
                       uint64_t cap_aln, uint64_t cap_ops, uint64_t cap_seq_bytes, uint32_t* contig, uint32_t* ref_start,
                       uint32_t* read_id, uint32_t* seq_off, uint16_t* seq_len, uint32_t* cigar_off, uint16_t* n_cigar, uint32_t* nm,
                       uint8_t* flags, uint32_t* cigar_ops, uint8_t* seq_pool,
                       uint64_t* counts /* in: aln, ops, blk, read bases; out: new totals; [4] = lines, [5] = first bad line */) {
    std::vector<std::string> nv;
    for (uint32_t i = 0; i < n_names; ++i) nv.emplace_back(names[i]);
    tok::TableImage im;
    tok::build_table_image(nv, im);
    const tok::ContigTable ct = tok::table_view(im, im.bytes.data());
    const uint8_t* nibtab = im.bytes.data() + im.o_nib;
    // padded, 8-byte aligned copy of the text (what ctx->b[B_TEXT] holds)
    std::vector<uint64_t> buf((n + 15) / 8 + 8, 0);
    uint8_t* text = reinterpret_cast<uint8_t*>(buf.data());
    memcpy(text, text_in, n);
    const bool unterminated = n > 0 && text[n - 1] != '\n';
    std::vector<uint64_t> line_start{0};
    for (uint64_t p = 0; p < n; ++p) if (text[p] == '\n') line_start.push_back(p + 1);
    const uint64_t n_lines = line_start.size() - 1 + (unterminated ? 1 : 0);
    counts[4] = n_lines;
    counts[5] = ~0ull;
    if (n_lines == 0) return PP_TOK_HOST;
    std::vector<tok::LineRec> recs(n_lines);
    std::vector<uint64_t> s_al(n_lines + 1, 0), s_ops(n_lines + 1, 0), s_blk(n_lines + 1, 0);
    bool need8 = false;
    uint64_t first_bad = ~0ull;
    auto span = [&](uint64_t i, uint64_t& s, uint64_t& e) {
        s = line_start[i];
        if (i + 1 == n_lines && unterminated) { e = n; return; }
        e = line_start[i + 1] - 1;
        if (e > s && text[e - 1] == '\r') e--;
    };
    for (uint64_t i = 0; i < n_lines; ++i) {
        tok::Txt x(text);
        uint64_t s, e;
        span(i, s, e);
        tok::LineRec r;
        const uint8_t kind = tok::parse_line(x, s, e, ct, nibtab, r);
        r.kind = kind;
        recs[i] = r;
        const bool al = kind == tok::LK_ALIGNED;
        s_al[i] = al; s_ops[i] = al ? r.nops : 0; s_blk[i] = al ? tok::seq_blocks(r) : 0;
        if (kind == tok::LK_HOST && i < first_bad) first_bad = i;
        if (al && r.need8) need8 = true;
    }
    auto exscan = [](std::vector<uint64_t>& v) { uint64_t run = 0; for (auto& x : v) { uint64_t t = x; x = run; run += t; } };
    exscan(s_al); exscan(s_ops); exscan(s_blk);
    const uint64_t n_al = s_al[n_lines], n_ops = s_ops[n_lines], n_blk = s_blk[n_lines];
    counts[5] = first_bad;
    if (first_bad != ~0ull) return PP_TOK_HOST;
    if (n_al == 0) return PP_TOK_HOST;
    const uint64_t A0 = counts[0], O0 = counts[1], B0 = counts[2], R0 = counts[3];
    const uint64_t blk_bytes = bits == 4 ? 16 : 32;
    if (A0 + n_al > cap_aln || O0 + n_ops > cap_ops || (B0 + n_blk) * blk_bytes > cap_seq_bytes) return PP_ERR_ARG;
    std::vector<uint64_t> name_pos(n_al);
    std::vector<uint32_t> name_len(n_al), head(n_al), rs(n_al);
    for (uint64_t i = 0; i < n_lines; ++i) {
        const tok::LineRec& r = recs[i];
        if (r.kind != tok::LK_ALIGNED) continue;
        const uint64_t s = line_start[i], la = s_al[i], A = A0 + la, co = O0 + s_ops[i], bo = B0 + s_blk[i];
        const bool star = r.flags & PP_FLAG_SEQSTAR;
        contig[A] = r.contig; ref_start[A] = r.ref_start; seq_off[A] = star ? 0u : (uint32_t)bo; seq_len[A] = (uint16_t)r.slen;
        cigar_off[A] = (uint32_t)co; n_cigar[A] = (uint16_t)r.nops; nm[A] = r.nm; flags[A] = r.flags;
        name_pos[la] = s; name_len[la] = r.name_len;
        tok::Txt x(text);
        tok::emit_cigar(x, s, r, cigar_ops + co);
        if (bits == 4) { if (tok::emit_seq<4>(x, s, r, nibtab, seq_pool + bo * 16)) need8 = true; }
        else tok::emit_seq<8>(x, s, r, nibtab, seq_pool + bo * 32);
    }
    for (uint64_t a = 0; a < n_al; ++a) {
        tok::Txt x(text);
        head[a] = tok::group_head(x, a, 0, name_pos.data(), name_len.data()) ? 1u : 0u;
    }
    uint32_t run = 0;
    for (uint64_t a = 0; a < n_al; ++a) { run += head[a]; rs[a] = run; }
    bool group_err = false;
    for (uint64_t a = 0; a < n_al; ++a) {
        read_id[A0 + a] = (uint32_t)(R0 + rs[a] - 1);
        if (head[a] && !tok::close_group(a, n_al, head.data(), careful != 0, seq_off + A0, seq_len + A0, flags + A0)) group_err = true;
    }
    if (group_err) return PP_TOK_HOST;
    if (need8 && bits == 4) return PP_TOK_NEED8;
    counts[0] = A0 + n_al; counts[1] = O0 + n_ops; counts[2] = B0 + n_blk; counts[3] = R0 + rs[n_al - 1];
    return PP_OK;
}

// The quick parse of `polypolish filter` (tok_line.h parse_line_quick), line by line.
extern "C" int ftok_cpu(const char* text_in, uint64_t n, uint64_t cap_lines, uint8_t* kind, uint32_t* ref_start, uint32_t* ref_end, uint8_t* rev,
                        uint32_t* name_len, uint32_t* ref_rel, uint32_t* ref_len, uint64_t* name_hash, uint64_t* ref_hash, uint64_t* n_lines_out) {
    std::vector<uint64_t> buf((n + 15) / 8 + 8, 0);
    uint8_t* text = reinterpret_cast<uint8_t*>(buf.data());
    memcpy(text, text_in, n);
    const bool unterminated = n > 0 && text[n - 1] != '\n';
    std::vector<uint64_t> line_start{0};
    for (uint64_t p = 0; p < n; ++p) if (text[p] == '\n') line_start.push_back(p + 1);
    const uint64_t n_lines = line_start.size() - 1 + (unterminated ? 1 : 0);
    *n_lines_out = n_lines;
    if (n_lines > cap_lines) return -1;
    for (uint64_t i = 0; i < n_lines; ++i) {
        uint64_t s = line_start[i], e;
        if (i + 1 == n_lines && unterminated) e = n;
        else { e = line_start[i + 1] - 1; if (e > s && text[e - 1] == '\r') e--; }
        tok::Txt x(text);
        tok::FLineRec r;
        kind[i] = tok::parse_line_quick(x, s, e, r);
        ref_start[i] = r.ref_start; ref_end[i] = r.ref_end; rev[i] = r.rev; name_len[i] = r.name_len; ref_rel[i] = r.ref_rel; ref_len[i] = r.ref_len;
        name_hash[i] = r.name_hash; ref_hash[i] = r.ref_hash;
    }
    return 0;
}

// The contig table's key of a name (tok_table.h).
extern "C" uint64_t fnv1a_cpu(const char* s, uint64_t n) { return tok::fnv1a(std::string(s, (size_t)n)); }

// The upload-side QUAL stripping (tok_strip.h).
#include "../polypolish_b200/csrc/tok_strip.h"
extern "C" uint64_t strip_cpu(const char* src, uint64_t n, char* dst) {
    return tok::strip_qual_lines(reinterpret_cast<const uint8_t*>(src), (size_t)n, reinterpret_cast<uint8_t*>(dst));
}

// The stripping upload, emulated: the same slice logic as upload_file_stripped (tok_kernels.cu) with nominal slices of S bytes
// and a look-ahead of `look`, the copies applied to a host buffer.  Returns 0, or 3 when a line end is further than `look`.
extern "C" int upload_emulate(const char* text_in, uint64_t n, uint64_t S, uint64_t look, char* out, uint8_t* last_byte, uint64_t* sent) {
    const uint8_t* text = reinterpret_cast<const uint8_t*>(text_in);
    std::vector<uint8_t> pin(S + look + 16);
    memset(out, 0xEE, n);
    *sent = 0;
    const uint64_t n_slices = (n + S - 1) / S;
    for (uint64_t k = 0; k < n_slices; ++k) {
        const uint64_t o = k * S, e = std::min<uint64_t>(n, o + S);
        const uint64_t rd0 = k ? o - 1 : 0, rd1 = std::min<uint64_t>(n, e + look - 1);
        const tok::SliceOut so = tok::strip_slice(text + rd0, rd0, rd1, k, e, n, pin.data());
        if (so.status == 3) return 3;
        if (so.status == 1) continue;
        if (so.ends_file) *last_byte = so.last;
        tok::apply_slice(so, pin.data(), reinterpret_cast<uint8_t*>(out));
        *sent += so.c;
    }
    return 0;
}
