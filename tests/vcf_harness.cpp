// CPU harness for the records of `polish --vcf` (polypolish_b200/csrc/vcf_records.h), compiled by tests/test_vcf_cpu.py with g++.
// It writes the whole file the way host_api.cpp's write_vcf does: the header over every contig, then each contig's records.
#include <string.h>

#include <vector>

#include "../polypolish_b200/csrc/vcf_records.h"

extern "C" {

// contig c: names[c], draft[c] (len[c] bytes), its changed positions [first[c], first[c + 1]) of pos / allele / depth / support.
// Copies min(cap, size) bytes of the file to out and returns its size.
size_t h_vcf(uint32_t n_contigs, const char* const* names, const char* const* draft, const uint64_t* len, const uint64_t* first,
             const uint64_t* pos, const char* const* allele, const double* depth, const uint32_t* support, char* out, size_t cap) {
    std::string buf;
    pp::vcf_header_begin(buf);
    for (uint32_t c = 0; c < n_contigs; ++c) pp::vcf_header_contig(buf, names[c], len[c]);
    pp::vcf_header_end(buf);
    for (uint32_t c = 0; c < n_contigs; ++c) {
        std::vector<pp::VcfChange> ch;
        for (uint64_t i = first[c]; i < first[c + 1]; ++i) ch.push_back({pos[i], allele[i], depth[i], support[i]});
        pp::vcf_records(buf, names[c], (const uint8_t*)draft[c], len[c], ch.data(), ch.size());
    }
    memcpy(out, buf.data(), buf.size() < cap ? buf.size() : cap);
    return buf.size();
}
}
