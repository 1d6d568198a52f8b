// vcf_records.h — the records of `polish --vcf`: one contig's edits as VCF lines whose application to the draft gives the polished
// contig byte for byte.  Pure host code with no CUDA and no context, used by host_api.cpp and compiled on its own by
// tests/vcf_harness.cpp.
//
// out(p), what position p puts into the FASTA: the emitted allele when p's status is changed, else the draft character; a '-' counts
// as nothing either way (polish.rs:188 drops every '-').  The edited positions E are the changed ones and the draft's '-'.  Per
// maximal run [a, b] of E: REF = draft[a..=b], ALT = out(a) .. out(b); no record when ALT == REF.  An empty ALT takes a padding base,
// draft[a - 1] in front (POS = a), or at a contig start draft[b + 1] behind (POS = 1); a run over the whole contig is REF = the
// contig, ALT = <DEL>.  A run at the contig start padded behind and a next run starting at b + 2 with an empty ALT would share
// draft[b + 1]: the two runs and that base make one record.  No left-alignment or other normalisation.
#pragma once
#include <algorithm>
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <string>
#include <string_view>

namespace pp {

// one changed position of a contig: 0-based position, the allele it emits ("-" for a deletion), its --debug depth and the pileup
// count of that allele
struct VcfChange {
    uint64_t pos;
    std::string_view allele;
    double depth;
    uint32_t support;
};

inline void vcf_header_begin(std::string& buf) {
    buf += "##fileformat=VCFv4.2\n##source=polypolish-b200\n";
}

inline void vcf_header_contig(std::string& buf, const char* name, uint64_t length) {
    buf += "##contig=<ID="; buf += name; buf += ",length="; buf += std::to_string(length); buf += ">\n";
}

inline void vcf_header_end(std::string& buf) {
    buf += "##ALT=<ID=DEL,Description=\"Whole contig removed by polishing\">\n"
           "##INFO=<ID=CHANGED,Number=1,Type=Integer,Description=\"Positions in the record whose polish status is changed\">\n"
           "##INFO=<ID=DEPTH,Number=.,Type=Float,Description=\"Read depth of each changed position, as in the --debug depth column\">\n"
           "##INFO=<ID=SUPPORT,Number=.,Type=Integer,Description=\"Pileup count of the allele each changed position took\">\n"
           "#CHROM\tPOS\tID\tREF\tALT\tQUAL\tFILTER\tINFO\n";
}

// Appends the records of one contig: `draft` its `len` bytes, `ch[0..n)` its changed positions in increasing order.
inline void vcf_records(std::string& buf, const char* name, const uint8_t* draft, uint64_t len, const VcfChange* ch, size_t n) {
    const char* d = (const char*)draft;
    // the first '-' at or after p (len: none); p never decreases from call to call, so the draft is scanned once
    uint64_t dash = 0;
    bool dash_known = false;
    auto dash_from = [&](uint64_t p) -> uint64_t {
        if (!dash_known || dash < p) {
            const void* q = p < len ? memchr(d + p, '-', len - p) : nullptr;
            dash = q ? (uint64_t)((const char*)q - d) : len;
            dash_known = true;
        }
        return dash;
    };
    // the next run of E at or after p: [a, b) and its changes ch[k0, k1)
    struct Run { uint64_t a, b; size_t k0, k1; };
    auto next_run = [&](uint64_t p, size_t k) -> Run {
        const uint64_t a = std::min(dash_from(p), k < n ? ch[k].pos : len);
        Run r{a, a, k, k};
        while (r.b < len) {
            if (r.k1 < n && ch[r.k1].pos == r.b) ++r.k1;
            else if (d[r.b] != '-') break;
            ++r.b;
        }
        return r;
    };
    auto alt_of = [&](const Run& r) {
        std::string alt;
        size_t k = r.k0;
        for (uint64_t p = r.a; p < r.b; ++p) {
            if (k < r.k1 && ch[k].pos == p) {
                for (char c : ch[k++].allele) if (c != '-') alt += c;
            } else if (d[p] != '-') {
                alt += d[p];
            }
        }
        return alt;
    };
    char tmp[64];
    uint64_t p = 0;
    size_t k = 0;
    while (true) {
        Run r = next_run(p, k);
        if (r.a >= len) break;
        std::string alt = alt_of(r);
        if (alt.empty() && r.a == 0 && r.b < len) {
            const Run s = next_run(r.b, r.k1);
            if (s.a == r.b + 1 && s.a < len && alt_of(s).empty()) {      // both would take draft[r.b]: one record
                r.b = s.b; r.k1 = s.k1;
                alt = alt_of(r);
            }
        }
        p = r.b; k = r.k1;
        std::string ref(d + r.a, (size_t)(r.b - r.a));
        if (alt == ref) continue;
        uint64_t pos = r.a + 1;
        if (alt.empty()) {
            if (r.a > 0) { ref.insert(ref.begin(), d[r.a - 1]); alt = d[r.a - 1]; pos = r.a; }
            else if (r.b < len) { ref += d[r.b]; alt = d[r.b]; pos = 1; }
            else { alt = "<DEL>"; pos = 1; }
        }
        buf += name; buf += '\t'; buf += std::to_string(pos); buf += "\t.\t"; buf += ref; buf += '\t'; buf += alt;
        buf += "\t.\tPASS\tCHANGED="; buf += std::to_string(r.k1 - r.k0);
        if (r.k1 > r.k0) {
            buf += ";DEPTH=";
            for (size_t i = r.k0; i < r.k1; ++i) {
                snprintf(tmp, sizeof tmp, "%.1f", ch[i].depth);      // the --debug depth column's bytes (debug_rows.h)
                if (i > r.k0) buf += ',';
                buf += tmp;
            }
            buf += ";SUPPORT=";
            for (size_t i = r.k0; i < r.k1; ++i) {
                if (i > r.k0) buf += ',';
                buf += std::to_string(ch[i].support);
            }
        }
        buf += '\n';
    }
}

}  // namespace pp
