// fasta.cpp — host-side FASTA loader and small text utilities.
//
// Behavioural mirror of misc::load_fasta (reference src/misc.rs:38-167): gzip detected by the
// magic bytes 1f 8b (:81-99), lines split like Rust's lines(), blank lines skipped (:111), header =
// name up to the first Unicode whitespace + description (:118-120), sequence lines concatenated and
// ASCII-upper-cased (:114,129), then the checks of check_load_fasta (:56-75) with the same messages.
#include <zlib.h>

#include <cstdio>
#include <cstdlib>
#include <unordered_set>

#include <sys/stat.h>

#include "pp_internal.h"

namespace pp {

bool read_file(const std::string& path, std::string& out) {
    FILE* f = fopen(path.c_str(), "rb");
    if (!f) return false;
    std::string buf;
    size_t have = 0;
    if (fseek(f, 0, SEEK_END) == 0) {            // regular file: one read straight into the string
        const long sz = ftell(f);
        fseek(f, 0, SEEK_SET);
        if (sz > 0) {
            buf.resize((size_t)sz);
            have = fread(&buf[0], 1, (size_t)sz, f);
            buf.resize(have);
        }
    }
    char tmp[1 << 16];                           // whatever is left (pipes, files that grew)
    size_t n;
    while ((n = fread(tmp, 1, sizeof tmp, f)) > 0) buf.append(tmp, n);
    bool ok = !ferror(f);
    fclose(f);
    if (!ok) return false;
    out.swap(buf);
    return true;
}

bool read_gz_file(const std::string& path, std::string& out) {
    gzFile g = gzopen(path.c_str(), "rb");
    if (!g) return false;
    gzbuffer(g, 1 << 20);
    std::string buf;
    char tmp[1 << 16];
    int n;
    while ((n = gzread(g, tmp, sizeof tmp)) > 0) buf.append(tmp, (size_t)n);
    gzclose(g);
    if (n < 0) return false;
    out.swap(buf);
    return true;
}

bool file_exists(const std::string& path) {      // Path::exists (misc.rs:218-223): a stat, never an open (a FIFO would block / lose its writer)
    struct stat sb;
    return stat(path.c_str(), &sb) == 0;
}

uint64_t file_size(const std::string& path) {
    struct stat sb;
    return stat(path.c_str(), &sb) == 0 ? (uint64_t)sb.st_size : 0;
}

bool parse_uint(std::string_view s, uint64_t maxv, uint64_t& out) {
    size_t i = 0;
    if (i < s.size() && s[i] == '+') i++;
    if (i >= s.size()) return false;
    uint64_t v = 0;
    for (; i < s.size(); ++i) {
        unsigned d = (unsigned)(s[i] - '0');
        if (d > 9) return false;
        if (v > (maxv - d) / 10) return false;
        v = v * 10 + d;
    }
    out = v;
    return true;
}

static inline bool is_op_letter(char c) {
    switch (c) {
        case 'M': case 'I': case 'D': case 'N': case 'S': case 'H': case 'P': case '=': case 'X': return true;
        default: return false;
    }
}

bool cigar_ref_end(std::string_view s, uint64_t start, uint64_t& end) {
    uint64_t ref_end = start;
    size_t i = 0, n = s.size();
    while (i < n) {
        if (s[i] >= '0' && s[i] <= '9') {
            size_t j = i;
            uint64_t v = 0;
            bool ovf = false;
            while (j < n && s[j] >= '0' && s[j] <= '9') {
                uint64_t d = (uint64_t)(s[j] - '0');
                if (v > (~0ull - d) / 10) ovf = true;
                v = v * 10 + d;
                j++;
            }
            if (j < n && is_op_letter(s[j])) {
                if (ovf) return false;
                char c = s[j];
                if (c == 'M' || c == 'D' || c == 'N' || c == '=' || c == 'X') ref_end += v;
                i = j + 1;
            } else {
                i = j;
            }
        } else {
            i++;
        }
    }
    end = ref_end;
    return true;
}

AlignedBytes::~AlignedBytes() { free(p); }
void AlignedBytes::reserve(size_t want) {
    if (want <= cap) return;
    size_t nc = cap ? cap : (1 << 20);
    while (nc < want) nc += nc / 2 + 64;
    nc = (nc + 63) & ~size_t(63);
    void* q = nullptr;
    if (posix_memalign(&q, 64, nc) != 0) throw std::bad_alloc();
    if (n) memcpy(q, p, n);
    free(p);
    p = (uint8_t*)q;
    cap = nc;
}
void AlignedBytes::resize_zero(size_t want) {
    if (want > n) {
        reserve(want);
        memset(p + n, 0, want - n);
    }
    n = want;
}

// Byte length of the Unicode White_Space character starting at s[i] (Rust char::is_whitespace), else 0.
static size_t unicode_ws_len(std::string_view s, size_t i) {
    unsigned char c = (unsigned char)s[i];
    if (c == ' ' || (c >= 0x09 && c <= 0x0D)) return 1;
    if (c == 0xC2 && i + 1 < s.size()) {
        unsigned char d = (unsigned char)s[i + 1];
        if (d == 0x85 || d == 0xA0) return 2;
    }
    if (i + 2 < s.size()) {
        unsigned char d = (unsigned char)s[i + 1], e = (unsigned char)s[i + 2];
        if (c == 0xE1 && d == 0x9A && e == 0x80) return 3;
        if (c == 0xE2 && d == 0x80 && ((e >= 0x80 && e <= 0x8A) || e == 0xA8 || e == 0xA9 || e == 0xAF)) return 3;
        if (c == 0xE2 && d == 0x81 && e == 0x9F) return 3;
        if (c == 0xE3 && d == 0x80 && e == 0x80) return 3;
    }
    return 0;
}

}  // namespace pp

static void set_err(char* err, size_t cap, const std::string& m) {
    if (!err || !cap) return;
    size_t n = m.size() < cap - 1 ? m.size() : cap - 1;
    memcpy(err, m.data(), n);
    err[n] = 0;
}

extern "C" pp_fasta* pp_fasta_load(const char* path, char* err, size_t errcap) {
    std::string filename = path ? path : "";
    std::string q = "\"" + filename + "\"";
    FILE* f = fopen(filename.c_str(), "rb");
    if (!f) { set_err(err, errcap, "unable to open " + q); return nullptr; }
    unsigned char magic[2];
    size_t got = fread(magic, 1, 2, f);
    fclose(f);
    if (got != 2) { set_err(err, errcap, q + " is too small"); return nullptr; }
    bool gz = magic[0] == 31 && magic[1] == 139;
    std::string data;
    if (!(gz ? pp::read_gz_file(filename, data) : pp::read_file(filename, data))) {
        set_err(err, errcap, "unable to load " + q);
        return nullptr;
    }
    pp_fasta* fa = new pp_fasta();
    fa->bases.reserve(data.size());
    bool have_name = false, bad_format = false;
    std::string name, desc;
    uint64_t seq_start = 0;
    auto flush = [&]() {
        fa->names.push_back(name);
        fa->descriptions.push_back(desc);
        fa->off.push_back(seq_start);
    };
    pp::for_each_line(data.data(), data.size(), [&](std::string_view text) {
        if (text.empty()) return true;
        if (text[0] == '>') {
            if (have_name) flush();
            std::string_view rest = text.substr(1);
            size_t i = 0, wl = 0;
            while (i < rest.size() && (wl = pp::unicode_ws_len(rest, i)) == 0) i++;
            if (i < rest.size()) { name.assign(rest.substr(0, i)); desc.assign(rest.substr(i + wl)); }
            else { name.assign(rest); desc.clear(); }
            have_name = name.size() > 0;   // the reference tests name.len() > 0 (misc.rs:113,122)
            seq_start = fa->bases.size();
            return true;
        }
        if (!have_name) { bad_format = true; return false; }
        const size_t o = fa->bases.size(), len = text.size();
        fa->bases.resize(o + len);
        char* dst = &fa->bases[o];
        const char* src = text.data();
        for (size_t k = 0; k < len; ++k) {           // ASCII upper-casing, branch-free so that it vectorises
            const unsigned char c = (unsigned char)src[k];
            dst[k] = (char)(c - (((unsigned)(c - 'a') < 26u) << 5));
        }
        return true;
    });
    if (bad_format) { set_err(err, errcap, q + " is not correctly formatted"); delete fa; return nullptr; }
    if (have_name) flush();
    fa->off.push_back(fa->bases.size());
    size_t n = fa->names.size();
    // A header with an empty name followed by sequence lines is "not correctly formatted" above, exactly as in
    // the reference; an empty-named header with no sequence simply vanishes there too.
    if (n == 0) { set_err(err, errcap, q + " contains no sequences"); delete fa; return nullptr; }
    for (size_t i = 0; i < n; ++i) {
        if (fa->names[i].empty()) { set_err(err, errcap, q + " has an unnamed sequence"); delete fa; return nullptr; }
        if (fa->off[i + 1] == fa->off[i]) { set_err(err, errcap, q + " has an empty sequence"); delete fa; return nullptr; }
    }
    for (size_t i = 0; i < n; ++i) {
        if (!fa->index.emplace(fa->names[i], (uint32_t)i).second) {
            set_err(err, errcap, q + " has a duplicated name");
            delete fa;
            return nullptr;
        }
    }
    return fa;
}

extern "C" void pp_fasta_free(pp_fasta* f) { delete f; }

extern "C" void pp_fasta_view(const pp_fasta* f, pp_contigs* out) {
    out->n_contigs = (uint32_t)f->names.size();
    out->off = f->off.data();
    out->bases = (const uint8_t*)f->bases.data();
}

extern "C" const char* pp_fasta_name(const pp_fasta* f, uint32_t i) {
    return i < f->names.size() ? f->names[i].c_str() : "";
}
extern "C" const char* pp_fasta_description(const pp_fasta* f, uint32_t i) {
    return i < f->descriptions.size() ? f->descriptions[i].c_str() : "";
}
