// debug_rows.h — the one formatter of --debug and --changes rows: write_debug_header / write_debug_line (polish.rs:247-266) over
// get_debug_line / get_count_str (pileup.rs:137-166).  Used by host_api.cpp, and by the CPU emulation of the kernels (tests/emu)
// so that the emulated change rows are checked byte for byte against the reference's.
#pragma once
#include <algorithm>
#include <charconv>
#include <cstdint>
#include <cstdio>
#include <string>
#include <vector>

#include "../../include/pp_abi.h"

namespace pp {

inline const char* const DEBUG_HEADER = "name\tpos\tbase\tdepth\tinvalid\tvalid\tpileup\tstatus\tnew_base\n";

// The --debug depth column's text ("%.1f" of the depth) of a depth printed as `tenths` tenths (depth_tenths in polish_dev.cuh), with
// no floating point: tenths / 10, ".", tenths % 10.
inline void depth_text(std::string& buf, uint64_t tenths) {
    char t[24];
    char* e = std::to_chars(t, t + sizeof t, tenths / 10).ptr;
    *e++ = '.';
    *e++ = (char)('0' + tenths % 10);
    buf.append(t, e);
}

inline uint32_t get_u32(const uint8_t* p) { return p[0] | (uint32_t)p[1] << 8 | (uint32_t)p[2] << 16 | (uint32_t)p[3] << 24; }

struct DebugRows {
    std::vector<std::string> counts;    // (reused from row to row)

    // One row: contig `name`, 0-based position `pos` in it, the position's record and its allele strings as k_allele_strings
    // wrote them (null when the position has no other allele and emits no node).
    void add(std::string& buf, const char* name, uint64_t pos, const pp_debug_pos& r, const uint8_t* alleles) {
        static const char* STATUS[6] = {"low_depth", "none", "multiple", "too_close", "kept", "changed"};
        static const char* ACGT = "ACGT";
        counts.clear();
        for (int b = 0; b < 4; ++b) if (r.count[b]) counts.push_back(std::string(1, ACGT[b]) + "x" + std::to_string(r.count[b]));
        if (r.count[4]) counts.push_back("-x" + std::to_string(r.count[4]));
        if (r.count[5]) counts.push_back(std::string(1, (char)r.original) + "x" + std::to_string(r.count[5]));
        std::string emitted;
        if (alleles) {
            const uint32_t n = get_u32(alleles);
            const uint8_t* q = alleles + 4;
            for (uint32_t i = 0; i < n; ++i) {
                const uint32_t count = get_u32(q), len = get_u32(q + 4);
                counts.push_back(std::string((const char*)q + 8, len) + "x" + std::to_string(count));
                q += 8 + len;
            }
            emitted.assign((const char*)q + 4, get_u32(q));
        }
        std::sort(counts.begin(), counts.end());
        char tmp[64];
        buf += name; buf += '\t'; buf += std::to_string(pos); buf += '\t'; buf += (char)r.original; buf += '\t';
        snprintf(tmp, sizeof tmp, "%.1f", r.depth);          // Rust {:.1}: both round the exact binary value
        buf += tmp; buf += '\t'; buf += std::to_string(r.invalid_threshold); buf += '\t'; buf += std::to_string(r.valid_threshold); buf += '\t';
        for (size_t k = 0; k < counts.size(); ++k) { if (k) buf += ','; buf += counts[k]; }
        buf += '\t'; buf += STATUS[r.status < 6 ? r.status : 0]; buf += '\t';
        if (r.new_node != 0xFFFFFFFFu) buf += emitted; else buf += (char)r.new_char;
        buf += '\n';
    }
};

}  // namespace pp
