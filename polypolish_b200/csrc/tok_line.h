// tok_line.h — per-line / per-alignment / per-group logic of the device SAM tokeniser (SURVEY.md §8f-1).
//
// These are the bodies the kernels of tok_kernels.cu run, one item per thread.  They are host+device so that the same
// code is exercised on the CPU by tests/tok_harness.cpp against the host packer (sam_pack.cpp), which stays the
// normative text layer: whatever this code is not sure about is answered with LK_HOST and the host packer decides
// (result or the reference's error text).  What is restated here:
//   Alignment::new          reference src/alignment.rs:49-98   columns, FLAG/POS, NM / ZP tags
//   get_expanded_cigar      reference src/alignment.rs:325-346 validation (\d+[MIDNSHP=X] tokens or "*")
//   add_to_pileup           reference src/alignment.rs:238-263 '@'/empty skipping, unaligned skipping, grouping rule
//   process_one_read        reference src/alignment.rs:275-295 source sequence of SEQ="*" records
#pragma once
#include <stdint.h>
#include <string.h>

#include "../../include/pp_abi.h"

#ifdef __CUDACC__
#define TK_HD __host__ __device__ __forceinline__
#else
#define TK_HD inline
#endif

namespace tok {

enum : uint8_t { LK_SKIP = 0, LK_ALIGNED = 1, LK_HOST = 2 };

// Byte reader over the text with one cached aligned 8-byte word (the text buffer is 8-byte aligned and padded).
struct Txt {
    const uint8_t* t;
    uint64_t w, wpos;
    TK_HD explicit Txt(const uint8_t* text) : t(text), w(0), wpos(~0ull) {}
    TK_HD uint8_t at(uint64_t p) {
        const uint64_t q = p & ~7ull;
        if (q != wpos) {
            wpos = q;
#ifdef __CUDA_ARCH__
            w = __ldg(reinterpret_cast<const unsigned long long*>(t + q));
#else
            memcpy(&w, t + q, 8);
#endif
        }
        return (uint8_t)(w >> (8 * (p & 7)));
    }
    // Position of the first '\t' in [p, e), or e.  (Word-at-a-time searches - a 64-bit zero-byte test, per-byte SIMD compares on
    // the two halves - were measured slower on the device than this loop over the cached word.)
    TK_HD uint64_t find_tab(uint64_t p, uint64_t e) {
        while (p < e && at(p) != '\t') ++p;
        return p;
    }
};

// Contig names: open addressing on the FNV-1a hash of the name, confirmed byte by byte.
struct ContigTable {
    const uint64_t* hash;      // [mask+1]
    const uint32_t* slot;      // [mask+1] contig index + 1, 0 = empty
    const uint32_t* name_off;  // [n_contigs+1] into names
    const uint8_t* names;
    uint32_t mask;
};

constexpr uint64_t FNV_BASIS = 14695981039346656037ull, FNV_PRIME = 1099511628211ull;

struct alignas(8) LineRec {    // what the parse pass keeps of one text line (40 bytes)
    uint32_t contig, ref_start, nm, nops;
    uint32_t slen, cig_rel, seq_rel, name_len;
    uint32_t cig_len;
    uint8_t flags, kind, need8, pad;
};

TK_HD int op_code(uint8_t c) {
    switch (c) {
        case 'M': return PP_OP_M; case 'I': return PP_OP_I; case 'D': return PP_OP_D; case 'N': return PP_OP_N;
        case 'S': return PP_OP_S; case 'H': return PP_OP_H; case 'P': return PP_OP_P; case '=': return PP_OP_EQ;
        case 'X': return PP_OP_X; default: return -1;
    }
}

// Rust "123".parse::<uN>() of the field starting at p (optional '+', >= 1 digit, overflow is an error); fe = field end.
TK_HD bool field_uint(Txt& x, uint64_t p, uint64_t e, uint64_t maxv, uint64_t& v, uint64_t& fe) {
    uint64_t i = p;
    v = 0;
    if (i < e && x.at(i) == '+') ++i;
    bool any = false;
    for (; i < e; ++i) {
        const uint8_t c = x.at(i);
        if (c == '\t') break;
        const unsigned d = (unsigned)c - '0';
        if (d > 9) return false;
        if (v > (maxv - d) / 10) return false;
        v = v * 10 + d;
        any = true;
    }
    fe = i;
    return any;
}

TK_HD uint64_t field_end(Txt& x, uint64_t p, uint64_t e) { return x.find_tab(p, e); }

TK_HD uint8_t lower(uint8_t c) { return (c >= 'A' && c <= 'Z') ? (uint8_t)(c + 32) : c; }

// One text line [s, e) (newline and one trailing '\r' already removed).  nibtab: 256-entry BAM nibble table (0 = not
// representable in 4 bits).  Returns the line's kind; r is complete for LK_ALIGNED.
TK_HD uint8_t parse_line(Txt& x, uint64_t s, uint64_t e, const ContigTable& ct, const uint8_t* nibtab, LineRec& r) {
    r.contig = PP_CONTIG_UNKNOWN; r.ref_start = 0; r.nm = 0; r.nops = 0; r.slen = 0; r.cig_rel = 0; r.seq_rel = 0;
    r.name_len = 0; r.cig_len = 0; r.flags = 0; r.kind = LK_SKIP; r.need8 = 0; r.pad = 0;
    if (e == s || x.at(s) == '@') return LK_SKIP;                       // alignment.rs:241-242
    if (e - s >= 0x7FFFFFFFull) return LK_HOST;
    uint64_t p = s, fe, v;
    // 0 QNAME
    fe = field_end(x, p, e);
    if (fe == e) return LK_HOST;                                        // too few columns
    r.name_len = (uint32_t)(fe - p);
    p = fe + 1;
    // 1 FLAG
    if (!field_uint(x, p, e, 0xFFFFFFFFull, v, fe) || fe == e) return LK_HOST;
    const uint32_t sam_flags = (uint32_t)v;
    const bool aligned = (sam_flags & 4) == 0;
    p = fe + 1;
    // 2 RNAME (hashed while scanned)
    const uint64_t rn = p;
    uint64_t h = FNV_BASIS;
    for (fe = p; fe < e; ++fe) {
        const uint8_t c = x.at(fe);
        if (c == '\t') break;
        h = (h ^ c) * FNV_PRIME;
    }
    if (fe == e) return LK_HOST;
    const uint32_t rn_len = (uint32_t)(fe - rn);
    p = fe + 1;
    // 3 POS
    if (!field_uint(x, p, e, ~0ull, v, fe) || fe == e) return LK_HOST;
    const uint64_t rstart = v > 0 ? v - 1 : 0;                          // alignment.rs:58-61
    p = fe + 1;
    // 4 MAPQ
    fe = field_end(x, p, e);
    if (fe == e) return LK_HOST;
    p = fe + 1;
    // 5 CIGAR: "*" or \d+[MIDNSHP=X] tokens (alignment.rs:325-346)
    r.cig_rel = (uint32_t)(p - s);
    uint32_t nops = 0;
    {
        uint64_t i = p;
        if (i < e && x.at(i) == '*' && (i + 1 == e || x.at(i + 1) == '\t')) {
            i++;
        } else {
            while (i < e) {
                uint8_t c = x.at(i);
                if (c == '\t') break;
                uint64_t len = 0;
                uint32_t nd = 0;
                while ((unsigned)c - '0' <= 9u) {
                    if (len <= 0xFFFFFFFFull) len = len * 10 + (c - '0');
                    nd++;
                    i++;
                    if (i >= e) return LK_HOST;                         // digits at the end of the line
                    c = x.at(i);
                }
                if (nd == 0 || op_code(c) < 0) return LK_HOST;          // invalid CIGAR string
                if (len > 0xFFFFFFFFull) return LK_HOST;
                if (len > 0 && aligned) {
                    if (len >= (1ull << 28)) return LK_HOST;
                    nops++;
                }
                i++;
            }
        }
        fe = i;
    }
    if (fe == e) return LK_HOST;
    r.cig_len = (uint32_t)(fe - p);
    p = fe + 1;
    // 6 RNEXT, 7 PNEXT, 8 TLEN
    for (int k = 0; k < 3; ++k) {
        fe = field_end(x, p, e);
        if (fe == e) return LK_HOST;
        p = fe + 1;
    }
    // 9 SEQ (its alphabet is checked where the bases are converted: emit_seq)
    r.seq_rel = (uint32_t)(p - s);
    fe = field_end(x, p, e);
    if (fe == e) return LK_HOST;
    const uint64_t slen = fe - p;
    const bool star = slen == 1 && x.at(p) == '*';
    p = fe + 1;
    // 10 QUAL
    fe = field_end(x, p, e);
    // 11.. tags (alignment.rs:67-75): NM:i: (last wins), ZP:Z:fail (ASCII case-insensitive, whole field)
    uint32_t mismatches = 0xFFFFFFFFu;
    bool pass_qc = true;
    if (fe < e) {
        p = fe + 1;
        for (;;) {                                                       // p <= e: an empty last field is still a field
            const uint64_t te = field_end(x, p, e);
            const uint64_t tl = te - p;
            if (tl >= 5 && x.at(p) == 'N' && x.at(p + 1) == 'M' && x.at(p + 2) == ':' && x.at(p + 3) == 'i' && x.at(p + 4) == ':') {
                uint64_t nv, ne;
                if (!field_uint(x, p + 5, te, 0xFFFFFFFFull, nv, ne)) return LK_HOST;
                mismatches = (uint32_t)nv;
            }
            if (tl == 9 && lower(x.at(p)) == 'z' && lower(x.at(p + 1)) == 'p' && x.at(p + 2) == ':' && lower(x.at(p + 3)) == 'z' &&
                x.at(p + 4) == ':' && lower(x.at(p + 5)) == 'f' && lower(x.at(p + 6)) == 'a' && lower(x.at(p + 7)) == 'i' &&
                lower(x.at(p + 8)) == 'l')
                pass_qc = false;
            if (te >= e) break;
            p = te + 1;
        }
    }
    if (mismatches == 0xFFFFFFFFu && aligned) return LK_HOST;           // missing NM tag
    if (!aligned) return LK_SKIP;                                       // alignment.rs:250
    if (nops == 0 || nops > 0xFFFFu) return LK_HOST;
    if (rstart > 0xFFFFFFFEull) return LK_HOST;
    if (!star && slen > 0xFFFFu) return LK_HOST;
    // contig index of RNAME
    for (uint32_t sl = (uint32_t)h & ct.mask;; sl = (sl + 1) & ct.mask) {
        const uint32_t c1 = ct.slot[sl];
        if (c1 == 0) break;
        if (ct.hash[sl] != h) continue;
        const uint32_t o = ct.name_off[c1 - 1], l = ct.name_off[c1] - o;
        if (l != rn_len) continue;
        uint32_t k = 0;
        while (k < l && ct.names[o + k] == x.at(rn + k)) ++k;
        if (k == l) { r.contig = c1 - 1; break; }
    }
    r.ref_start = (uint32_t)rstart;
    r.nm = mismatches;
    r.nops = nops;
    r.slen = star ? 0 : (uint32_t)slen;
    r.flags = (uint8_t)(((sam_flags & 16) ? PP_FLAG_REVERSE : 0) | (pass_qc ? 0 : PP_FLAG_ZPFAIL) | (star ? PP_FLAG_SEQSTAR : 0));
    r.need8 = 0;
    r.kind = LK_ALIGNED;
    return LK_ALIGNED;
}

// 32-base blocks of one record's sequence.
TK_HD uint32_t seq_blocks(const LineRec& r) { return (r.flags & PP_FLAG_SEQSTAR) ? 0u : (r.slen + PP_SEQ_BLOCK - 1) / PP_SEQ_BLOCK; }

// Second visit of an aligned line: its CIGAR operations (len << 4 | op, zero-length operations dropped).
TK_HD void emit_cigar(Txt& x, uint64_t s, const LineRec& r, uint32_t* ops) {
    uint64_t i = s + r.cig_rel;
    const uint64_t e = i + r.cig_len;
    uint32_t k = 0;
    while (i < e && k < r.nops) {
        uint64_t len = 0;
        uint8_t c = x.at(i);
        while ((unsigned)c - '0' <= 9u) { len = len * 10 + (c - '0'); c = x.at(++i); }
        if (len > 0) ops[k++] = (uint32_t)(len << 4) | (uint32_t)op_code(c);
        i++;
    }
}

// ... and its sequence: 4-bit BAM codes (16 bytes per block) or upper-cased bytes (32 bytes per block), zero padded.
// Returns true (4-bit pool only) when a base has no 4-bit code: the pool must be rebuilt with 8-bit bases.
template <int BITS>
TK_HD bool emit_seq(Txt& x, uint64_t s, const LineRec& r, const uint8_t* nibtab, uint8_t* dst) {
    const uint64_t b = s + r.seq_rel;
    const uint32_t n = r.slen, nblk = seq_blocks(r);
    bool exotic = false;
    for (uint32_t blk = 0; blk < nblk; ++blk) {
        if (BITS == 4) {
            uint64_t lo = 0, hi = 0;
            for (uint32_t j = 0; j < 16; ++j) {
                const uint32_t q = blk * 32 + j;
                if (q < n) { const uint8_t c = nibtab[x.at(b + q)]; exotic |= c == 0; lo |= (uint64_t)c << (4 * j); }
            }
            for (uint32_t j = 0; j < 16; ++j) {
                const uint32_t q = blk * 32 + 16 + j;
                if (q < n) { const uint8_t c = nibtab[x.at(b + q)]; exotic |= c == 0; hi |= (uint64_t)c << (4 * j); }
            }
            uint64_t* d = reinterpret_cast<uint64_t*>(dst + (size_t)blk * 16);
            d[0] = lo; d[1] = hi;
        } else {
            for (uint32_t w = 0; w < 4; ++w) {
                uint64_t v = 0;
                for (uint32_t j = 0; j < 8; ++j) {
                    const uint32_t q = blk * 32 + w * 8 + j;
                    if (q < n) {
                        uint8_t c = x.at(b + q);
                        if (c >= 'a' && c <= 'z') c = (uint8_t)(c - 32);
                        v |= (uint64_t)c << (8 * j);
                    }
                }
                reinterpret_cast<uint64_t*>(dst + (size_t)blk * 32)[w] = v;
            }
        }
    }
    return exotic;
}

// Does alignment a open a new read group?  (alignment.rs:255: a record joins the open group iff the open name is empty
// or equals its QNAME; every file starts with no open group.)
TK_HD bool group_head(Txt& x, uint64_t a, uint64_t file_first, const uint64_t* name_pos, const uint32_t* name_len) {
    if (a == file_first) return true;
    const uint32_t lp = name_len[a - 1], lc = name_len[a];
    if (lp == 0) return false;
    if (lp != lc) return true;
    const uint64_t pp = name_pos[a - 1], pc = name_pos[a];
    Txt y(x.t);
    for (uint32_t k = 0; k < lp; ++k)
        if (x.at(pp + k) != y.at(pc + k)) return true;
    return false;
}

// Closes the group whose first alignment is a (run by the thread of every group head): SEQ="*" records take the group's
// source sequence, the first record with a sequence (alignment.rs:311-318), reverse-complemented when the strands differ
// (alignment.rs:290-295).  Returns false for the reference's "no alignments for read ... contain sequence" case.
TK_HD bool close_group(uint64_t a, uint64_t file_end, const uint32_t* head, bool careful, uint32_t* seq_off, uint16_t* seq_len, uint8_t* flags) {
    uint64_t b = a, src = ~0ull;
    do {
        if (src == ~0ull && !(flags[b] & PP_FLAG_SEQSTAR)) src = b;
        ++b;
    } while (b < file_end && !head[b]);
    const uint64_t n = b - a;
    const bool skipped = careful && n > 1;                              // alignment.rs:277-279
    if (src == ~0ull && !skipped) return false;
    for (uint64_t c = a; c < b; ++c) {
        if (!(flags[c] & PP_FLAG_SEQSTAR)) continue;
        if (src != ~0ull) {
            seq_off[c] = seq_off[src];
            seq_len[c] = seq_len[src];
            if ((flags[c] ^ flags[src]) & PP_FLAG_REVERSE) flags[c] |= PP_FLAG_RC;
        } else {
            flags[c] |= PP_FLAG_NOSEQ;
        }
    }
    return true;
}


// ---- `polypolish filter`: the quick parse (Alignment::new_quick alignment.rs:102-128 as used by filter.rs:110-145) ----------
enum : uint8_t { FK_VERBATIM = 0, FK_ALIGNED = 1, FK_HOST = 2 };   // header / unaligned line; keyed record; host decides

struct alignas(8) FLineRec {   // 40 bytes
    uint64_t name_hash, ref_hash;          // FNV-1a of QNAME / RNAME (interned on the device, confirmed byte by byte)
    uint32_t name_len, ref_rel, ref_len;   // QNAME starts the line; RNAME at ref_rel
    uint32_t ref_start, ref_end;           // 0-based start; get_ref_end (alignment.rs:138-149)
    uint8_t rev, kind, pad[2];
};

TK_HD bool is_ref_op(uint8_t c) { return c == 'M' || c == 'D' || c == 'N' || c == '=' || c == 'X'; }

// Alignment::get_ref_end: tolerant scan of \d+[MIDNSHP=X] tokens in [p, fe); false when a token's length overflows u64.
TK_HD bool cigar_ref_end(Txt& x, uint64_t p, uint64_t fe, uint64_t start, uint64_t& end) {
    uint64_t ref_end = start, i = p;
    while (i < fe) {
        uint8_t c = x.at(i);
        if ((unsigned)c - '0' <= 9u) {
            uint64_t j = i, v = 0;
            bool ovf = false;
            while (j < fe && (unsigned)(c = x.at(j)) - '0' <= 9u) {
                const uint64_t d = c - '0';
                if (v > 1844674407370955160ull && v > (~0ull - d) / 10) ovf = true;
                v = v * 10 + d;
                j++;
            }
            if (j < fe && op_code(x.at(j)) >= 0) {
                if (ovf) return false;
                if (is_ref_op(x.at(j))) ref_end += v;
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

// One text line [s, e) of a SAM file given to `polypolish filter` (filter.rs:122-137): '@' lines are headers; every other
// line needs 11 columns, a FLAG and a POS; unaligned records are passed through; aligned ones are keyed by QNAME.
TK_HD uint8_t parse_line_quick(Txt& x, uint64_t s, uint64_t e, FLineRec& r) {
    r.name_hash = 0; r.ref_hash = 0; r.name_len = 0; r.ref_rel = 0; r.ref_len = 0; r.ref_start = 0; r.ref_end = 0;
    r.rev = 0; r.kind = FK_VERBATIM; r.pad[0] = r.pad[1] = 0;
    if (e > s && x.at(s) == '@') return FK_VERBATIM;
    if (e - s >= 0x7FFFFFFFull) return FK_HOST;
    uint64_t p = s, fe, v;
    // 0 QNAME
    uint64_t h = FNV_BASIS;
    for (fe = p; fe < e; ++fe) {
        const uint8_t c = x.at(fe);
        if (c == '\t') break;
        h = (h ^ c) * FNV_PRIME;
    }
    if (fe == e) return FK_HOST;                                        // too few columns (an empty line too)
    r.name_hash = h;
    r.name_len = (uint32_t)(fe - p);
    p = fe + 1;
    // 1 FLAG
    if (!field_uint(x, p, e, 0xFFFFFFFFull, v, fe) || fe == e) return FK_HOST;
    const uint32_t sam_flags = (uint32_t)v;
    p = fe + 1;
    // 2 RNAME
    r.ref_rel = (uint32_t)(p - s);
    h = FNV_BASIS;
    for (fe = p; fe < e; ++fe) {
        const uint8_t c = x.at(fe);
        if (c == '\t') break;
        h = (h ^ c) * FNV_PRIME;
    }
    if (fe == e) return FK_HOST;
    r.ref_hash = h;
    r.ref_len = (uint32_t)(fe - p);
    p = fe + 1;
    // 3 POS
    if (!field_uint(x, p, e, ~0ull, v, fe) || fe == e) return FK_HOST;
    const uint64_t start = v > 0 ? v - 1 : 0;
    p = fe + 1;
    // 4 MAPQ
    fe = field_end(x, p, e);
    if (fe == e) return FK_HOST;
    p = fe + 1;
    // 5 CIGAR
    const uint64_t cg = p;
    fe = field_end(x, p, e);
    if (fe == e) return FK_HOST;
    const uint64_t cg_end = fe;
    p = fe + 1;
    // 6..9 must exist (column 10 may be the last)
    for (int k = 0; k < 4; ++k) {
        fe = field_end(x, p, e);
        if (fe == e) return FK_HOST;
        p = fe + 1;
    }
    if (sam_flags & 4) return FK_VERBATIM;                              // filter.rs:132
    uint64_t end;
    if (!cigar_ref_end(x, cg, cg_end, start, end) || end > 0xFFFFFFFEull) return FK_HOST;
    r.ref_start = (uint32_t)start;
    r.ref_end = (uint32_t)end;
    r.rev = (sam_flags & 16) ? 1 : 0;
    r.kind = FK_ALIGNED;
    return FK_ALIGNED;
}

// Do two byte ranges of the text(s) hold the same string?
TK_HD bool same_bytes(Txt& a, uint64_t pa, Txt& b, uint64_t pb, uint32_t len) {
    for (uint32_t k = 0; k < len; ++k)
        if (a.at(pa + k) != b.at(pb + k)) return false;
    return true;
}

}  // namespace tok
