// host_api.cpp — whole-command drivers above the C-ABI compute calls.
//
// Mirrors the reference's command drivers (same option checks, same error text, same stdout bytes):
//   polish::polish            reference src/polish.rs:26-38   (+ :93-134 loading, :137-203 output)
//   filter::filter            reference src/filter.rs:26-37   (+ :273-349 SAM re-streaming)
// Text (FASTA/SAM) is handled here on the host; all per-alignment / per-position work is behind
// pp_polish() / pp_filter() on the device.  There is no CPU fallback for that work.
#include <chrono>
#include <cmath>
#include <fcntl.h>
#include <sys/stat.h>
#include <unistd.h>
#include <cstdio>
#include <cstdlib>
#include <algorithm>
#include <memory>
#include <string>
#include <thread>
#include <utility>
#include <vector>

#include "pp_internal.h"

namespace {

std::string fmt_thousands(uint64_t v) {      // num_format Locale::en
    std::string s = std::to_string(v), o;
    int n = (int)s.size();
    for (int i = 0; i < n; ++i) {
        o += s[i];
        if ((n - 1 - i) % 3 == 0 && i != n - 1) o += ',';
    }
    return o;
}

// polish.rs:290-300 qscore: "Q∞" at 100 %, "Q0" at or below 0 %, else Q{-10 log10(1 - identity/100)} with two decimals
std::string qscore_text(double identity) {
    if (identity >= 100.0) return "Q\xe2\x88\x9e";
    if (identity <= 0.0) return "Q0";
    const double errors = 1.0 - (identity / 100.0);
    char tmp[64];
    snprintf(tmp, sizeof tmp, "Q%.2f", -10.0 * std::log10(errors));
    return tmp;
}

}  // namespace

extern "C" void pp_free(void* p) { free(p); }

// misc.rs:170-182 complement_base (upper-case input)
static char complement_char(char b) {
    switch (b) {
        case 'A': return 'T'; case 'T': return 'A'; case 'G': return 'C'; case 'C': return 'G'; case 'N': return 'N';
        case 'R': return 'Y'; case 'Y': return 'R'; case 'S': return 'S'; case 'W': return 'W'; case 'K': return 'M'; case 'M': return 'K';
        case 'B': return 'V'; case 'V': return 'B'; case 'D': return 'H'; case 'H': return 'D';
        case '.': return '.'; case '-': return '-'; case '?': return '?';
        default: return 'N';
    }
}

// The string of one "other" allele node (pileup.rs:62 key).
static std::string node_allele(const pp_debug_node& nd, const pp_alignments* a) {
    static const char* NIB = "=ACMGRSVTWYHKDBN";
    std::string out;
    if (a->seq_bits == 4 && (nd.sig & 15)) {
        for (uint32_t i = 0; i < (nd.sig & 15); ++i) out += NIB[(nd.sig >> (4 * (i + 1))) & 15];
        return out;
    }
    if (a->seq_bits == 8 && (nd.sig & 255)) {
        for (uint32_t i = 0; i < (nd.sig & 255); ++i) out += (char)((nd.sig >> (8 * (i + 1))) & 255);
        return out;
    }
    const uint32_t aln = (uint32_t)(nd.val >> 32), start = (uint32_t)(nd.val >> 16) & 0xFFFFu, len = (uint32_t)nd.val & 0xFFFFu;
    const bool rc = a->flags[aln] & PP_FLAG_RC;
    const uint32_t n = a->seq_len[aln];
    for (uint32_t i = 0; i < len; ++i) {
        const uint32_t e = start + i, j = rc ? (n - 1 - e) : e;
        char ch;
        if (a->seq_bits == 4) {
            const uint8_t b = a->seq_pool[(size_t)a->seq_off[aln] * (PP_SEQ_BLOCK / 2) + (j >> 1)];
            ch = NIB[(b >> ((j & 1) * 4)) & 15];
        } else {
            ch = (char)a->seq_pool[(size_t)a->seq_off[aln] * PP_SEQ_BLOCK + j];
        }
        out += rc ? complement_char(ch) : ch;
    }
    return out;
}

// write_debug_header / write_debug_line (polish.rs:247-266) + get_debug_line / get_count_str (pileup.rs:137-166)
static int write_debug_tsv(pp_ctx* ctx, const pp_fasta* fa, const pp_contigs* contigs, const pp_alignments* alns, FILE* f) {
    static const char* STATUS[6] = {"low_depth", "none", "multiple", "too_close", "kept", "changed"};
    const uint64_t G = contigs->off[contigs->n_contigs];
    std::vector<uint32_t> head(G);
    uint64_t n_nodes = 0;
    pp_polish_debug_alleles(ctx, nullptr, nullptr, 0, &n_nodes);           // size query (reports the node count, then fails on the null buffers)
    std::vector<pp_debug_node> nodes(n_nodes + 1);
    int rc = pp_polish_debug_alleles(ctx, head.data(), nodes.data(), n_nodes, &n_nodes);
    if (rc != PP_OK) return rc;
    if (fputs("name\tpos\tbase\tdepth\tinvalid\tvalid\tpileup\tstatus\tnew_base\n", f) < 0) return PP_ERR_IO;
    const uint64_t CH = 1 << 18;
    std::vector<pp_debug_pos> recs(CH);
    std::string buf;
    std::vector<std::string> counts;
    char tmp[64];
    for (uint32_t c = 0; c < contigs->n_contigs; ++c) {
        const char* name = pp_fasta_name(fa, c);
        for (uint64_t p0 = contigs->off[c]; p0 < contigs->off[c + 1]; p0 += CH) {
            const uint64_t n = std::min<uint64_t>(CH, contigs->off[c + 1] - p0);
            rc = pp_polish_debug_fetch(ctx, p0, n, recs.data());
            if (rc != PP_OK) return rc;
            buf.clear();
            for (uint64_t i = 0; i < n; ++i) {
                const pp_debug_pos& r = recs[i];
                const uint64_t gp = p0 + i;
                counts.clear();
                static const char* ACGT = "ACGT";
                for (int b = 0; b < 4; ++b) if (r.count[b]) counts.push_back(std::string(1, ACGT[b]) + "x" + std::to_string(r.count[b]));
                if (r.count[4]) counts.push_back("-x" + std::to_string(r.count[4]));
                if (r.count[5]) counts.push_back(std::string(1, (char)r.original) + "x" + std::to_string(r.count[5]));
                for (uint32_t nd = head[gp]; nd != 0;) {
                    const pp_debug_node& node = nodes[nd - 1];
                    counts.push_back(node_allele(node, alns) + "x" + std::to_string(node.count));
                    nd = node.next == 0xFFFFFFFFu ? 0 : node.next + 1;
                }
                std::sort(counts.begin(), counts.end());
                buf += name; buf += '\t'; buf += std::to_string(gp - contigs->off[c]); buf += '\t'; buf += (char)r.original; buf += '\t';
                snprintf(tmp, sizeof tmp, "%.1f", r.depth);          // Rust {:.1}: both round the exact binary value
                buf += tmp; buf += '\t'; buf += std::to_string(r.invalid_threshold); buf += '\t'; buf += std::to_string(r.valid_threshold); buf += '\t';
                for (size_t k = 0; k < counts.size(); ++k) { if (k) buf += ','; buf += counts[k]; }
                buf += '\t'; buf += STATUS[r.status < 6 ? r.status : 0]; buf += '\t';
                if (r.new_node != 0xFFFFFFFFu) buf += node_allele(nodes[r.new_node], alns); else buf += (char)r.new_char;
                buf += '\n';
            }
            if (fwrite(buf.data(), 1, buf.size(), f) != buf.size()) return PP_ERR_IO;
        }
    }
    return PP_OK;
}

// One shard on one GPU (run by its own host thread when there are several).
struct ShardJob {
    pp_ctx* ctx = nullptr;
    pp_contigs contigs;
    pp_alignments alns;
    const uint32_t* contig_map = nullptr;
    bool resident = false;               // the dataset is already on the device (device tokeniser)
    std::vector<uint64_t> out_off, changed, zero;
    std::vector<double> tdepth;
    std::vector<uint8_t> bases;
    pp_polish_result res;
    int rc = PP_OK;
    std::string err;
    // a shard made on the device (every GPU tokenises the text itself): the shard's contigs live here
    std::vector<uint32_t> own_map, own_local;
    std::vector<uint64_t> own_off;
    std::vector<uint8_t> own_bases;
};

static void run_shard(ShardJob* j, const pp_polish_params* prm) {
    const uint64_t G = j->contigs.off[j->contigs.n_contigs];
    j->out_off.assign(j->contigs.n_contigs + 1, 0);
    j->changed.assign(j->contigs.n_contigs, 0);
    j->zero.assign(j->contigs.n_contigs, 0);
    j->tdepth.assign(j->contigs.n_contigs, 0.0);
    memset(&j->res, 0, sizeof j->res);
    // Output is at most G + inserted bases; start with G + 1 MiB and retry once with the exact size.
    uint64_t cap = G + (1u << 20);
    for (int attempt = 0; attempt < 2; ++attempt) {
        j->bases.resize(cap);
        j->res.out_off = j->out_off.data();
        j->res.out_bases = j->bases.data();
        j->res.out_cap = cap;
        j->res.changed = j->changed.data();
        j->res.zero_depth = j->zero.data();
        j->res.total_depth = j->tdepth.data();
        j->rc = j->resident ? pp_polish_resident(j->ctx, prm, &j->res) : pp_polish(j->ctx, &j->contigs, &j->alns, prm, &j->res);
        if (j->rc == PP_ERR_ARG && j->res.out_len > cap) { cap = j->res.out_len; continue; }
        break;
    }
    if (j->rc != PP_OK) j->err = pp_last_error(j->ctx);
}

// The resident dataset of a context copied back into host arrays (pp_dataset_download).  Plain new[] without value
// initialisation: the copy overwrites every byte, so zero-filling 0.4 GB first would only cost time.
struct HostCopy {
    std::unique_ptr<uint32_t[]> contig, ref_start, read_id, seq_off, cigar_off, nm, cigar_ops;
    std::unique_ptr<uint16_t[]> seq_len, n_cigar;
    std::unique_ptr<uint8_t[]> flags, seq_pool;
    int fetch(pp_ctx* ctx, pp_alignments* v) {
        int rc = pp_dataset_sizes(ctx, v);
        if (rc != PP_OK) return rc;
        const size_t n = (size_t)v->n_aln + 1;
        contig.reset(new uint32_t[n]); ref_start.reset(new uint32_t[n]); read_id.reset(new uint32_t[n]); seq_off.reset(new uint32_t[n]);
        cigar_off.reset(new uint32_t[n]); nm.reset(new uint32_t[n]); seq_len.reset(new uint16_t[n]); n_cigar.reset(new uint16_t[n]);
        flags.reset(new uint8_t[n]); cigar_ops.reset(new uint32_t[(size_t)v->n_cigar_ops + 1]); seq_pool.reset(new uint8_t[(size_t)v->seq_pool_bytes + 64]);
        v->contig = contig.get(); v->ref_start = ref_start.get(); v->read_id = read_id.get(); v->seq_off = seq_off.get();
        v->cigar_off = cigar_off.get(); v->nm = nm.get(); v->seq_len = seq_len.get(); v->n_cigar = n_cigar.get(); v->flags = flags.get();
        v->cigar_ops = cigar_ops.get(); v->seq_pool = seq_pool.get();
        return pp_dataset_download(ctx, v);
    }
};

// SAM files -> resident dataset through the device tokeniser (tok_kernels.cu).  PP_OK, PP_TOK_HOST (the host packer must
// look at the text), or an error.  `log` collects the per-file lines add_to_pileup prints (alignment.rs:266-271).
// Cuts a SAM file into n byte ranges for n GPUs: cut[0] = 0, cut[n] = size, every other cut is the start of a line whose QNAME differs from
// the line before it (a read group - consecutive lines of one QNAME, alignment.rs:214-272 - is never split).  false: not a plain file,
// or a line longer than the window (the caller lets one GPU read the whole file instead).
static bool split_ranges(const char* path, int n, std::vector<uint64_t>& cut) {
    const int fd = open(path, O_RDONLY);
    if (fd < 0) return false;
    struct stat sb;
    if (fstat(fd, &sb) != 0 || !S_ISREG(sb.st_mode)) { close(fd); return false; }
    const uint64_t S = (uint64_t)sb.st_size;
    cut.assign((size_t)n + 1, S);
    cut[0] = 0;
    const size_t W = 1 << 20;
    std::vector<char> buf(W);
    bool ok = true;
    // the line starting at `pos` (a line start): its QNAME and where the next line starts
    auto line_at = [&](uint64_t pos, std::string& qname, uint64_t& next) -> bool {
        if (pos >= S) return false;
        const size_t want = (size_t)std::min<uint64_t>(W, S - pos);
        size_t got = 0;
        while (got < want) {
            const ssize_t r = pread(fd, buf.data() + got, want - got, (off_t)(pos + got));
            if (r <= 0) { ok = false; return false; }
            got += (size_t)r;
        }
        const char* nl = (const char*)memchr(buf.data(), '\n', got);
        if (!nl && pos + got < S) { ok = false; return false; }                  // longer than the window
        const size_t len = nl ? (size_t)(nl - buf.data()) : got;
        const char* tab = (const char*)memchr(buf.data(), '\t', len);
        qname.assign(buf.data(), tab ? (size_t)(tab - buf.data()) : len);
        next = pos + len + 1;
        return true;
    };
    for (int g = 1; g < n && ok; ++g) {
        uint64_t pos = std::max<uint64_t>(S / (uint64_t)n * (uint64_t)g, cut[g - 1]);
        if (pos >= S) { cut[g] = S; continue; }
        // the first line start at or after pos
        if (pos > 0) {
            std::string q; uint64_t nx = 0;
            if (!line_at(pos - 1, q, nx)) { if (!ok) break; cut[g] = S; continue; }       // (the rest of the line that holds byte pos - 1)
            pos = std::min(nx, S);
        }
        // ... then on to the first line whose QNAME differs from its predecessor's
        std::string qa, qb;
        uint64_t na = 0, nb = 0;
        if (!line_at(pos, qa, na)) { if (!ok) break; cut[g] = S; continue; }
        uint64_t cand = std::min(na, S);
        for (;;) {
            if (cand >= S || !line_at(cand, qb, nb)) { cand = S; break; }
            if (qb != qa || (!qb.empty() && qb[0] == '@')) break;
            qa.swap(qb);
            cand = std::min(nb, S);
        }
        if (!ok) break;
        cut[g] = std::max(cand, cut[g - 1]);
    }
    close(fd);
    return ok;
}

extern "C" int pp_sam_split_ranges(const char* path, int n, uint64_t* cuts) {
    if (!path || n < 1 || !cuts) return PP_ERR_ARG;
    std::vector<uint64_t> c;
    if (!split_ranges(path, n, c)) return PP_ERR_IO;
    std::copy(c.begin(), c.end(), cuts);
    return PP_OK;
}

struct DeviceShard { const uint32_t* local_of; uint32_t n_total; pp_contigs contigs; bool takes_unknown; };
static int tokenise_files(pp_ctx* ctx, const pp_fasta* fa, const char* const* sams, int n_sams, bool careful, std::string& log,
                          std::string& timing, uint64_t* n_aln, const DeviceShard* shard = nullptr) {
    int bits = 4;
    for (int attempt = 0; attempt < 2; ++attempt) {
        log.clear(); timing.clear();
        *n_aln = 0;
        int rc = pp_tok_begin(ctx, fa, careful ? 1 : 0, bits);
        uint64_t total = 0;
        for (int i = 0; i < n_sams; ++i) total += pp::file_size(sams[i]);
        if (rc == PP_OK) rc = pp_tok_expect(ctx, total);
        if (rc == PP_OK && shard) rc = pp_tok_set_shard(ctx, shard->local_of, shard->n_total, &shard->contigs, shard->takes_unknown ? 1 : 0);
        std::vector<pp_tok_stats> st((size_t)n_sams);
        if (rc == PP_OK) rc = pp_tok_add_files(ctx, sams, n_sams, st.data());
        for (int i = 0; i < n_sams && rc == PP_OK; ++i) {
            *n_aln += st[i].alignments;
            log += std::string(sams[i]) + ": " + fmt_thousands(st[i].alignments) + " alignments from " + fmt_thousands(st[i].reads) + " reads\n";
            char tmp[256];
            snprintf(tmp, sizeof tmp, "SAM tokeniser %s: %s lines, text to HBM %.3f ms, %u kernels %.3f ms\n", sams[i], fmt_thousands(st[i].lines).c_str(),
                     st[i].h2d_ms, st[i].launches, st[i].device_ms);
            timing += tmp;
        }
        if (rc == PP_TOK_NEED8 && bits == 4) { bits = 8; continue; }
        if (rc == PP_TOK_NEED8) rc = PP_TOK_HOST;
        if (rc == PP_OK) rc = pp_tok_finish(ctx);
        return rc;
    }
    return PP_TOK_HOST;
}

// `filter` in front of `polish` in the same call (pp_filter_polish_files): the two SAM files are `sams`, this says what to filter with
struct FusedFilter {
    pp_filter_params prm;
    std::string orientation;
    const char *out1, *out2;             // filtered SAM files, or null: not written
};

// polish::polish (polish.rs:26-38) over one or several GPUs (contigs shard across them, SURVEY.md §8e).
static int polish_files_impl(pp_ctx* const* ctxs, int n_ctx, const char* assembly, const char* const* sams, int n_sams,
                             const pp_polish_params* prm, const char* debug_path, char** out_fasta, uint64_t* out_len, int verbose,
                             const FusedFilter* ff = nullptr) {
    pp_ctx* ctx = ctxs[0];
    if (!assembly || !prm || !out_fasta || !out_len || n_sams < 0) return pp_ctx_fail(ctx, PP_ERR_ARG, "pp_polish_files: bad arguments");
    *out_fasta = nullptr;
    *out_len = 0;
    // check_option_values polish.rs:277-287
    if (!(prm->fraction_valid > 0.0 && prm->fraction_valid < 1.0)) return pp_ctx_fail(ctx, PP_ERR_INPUT, "--fraction_valid must be between 0 and 1 (exclusive)");
    if (!(prm->fraction_invalid > 0.0 && prm->fraction_invalid < 1.0)) return pp_ctx_fail(ctx, PP_ERR_INPUT, "--fraction_invalid must be between 0 and 1 (exclusive)");
    if (prm->fraction_invalid >= prm->fraction_valid) return pp_ctx_fail(ctx, PP_ERR_INPUT, "--fraction_invalid must be less than --fraction_valid");
    // check_inputs_exist polish.rs:269-274
    if (!pp::file_exists(assembly)) return pp_ctx_fail(ctx, PP_ERR_INPUT, ("\"" + std::string(assembly) + "\" file does not exist").c_str());
    for (int i = 0; i < n_sams; ++i)
        if (!pp::file_exists(sams[i])) return pp_ctx_fail(ctx, PP_ERR_INPUT, ("\"" + std::string(sams[i]) + "\" file does not exist").c_str());
    const bool debug = debug_path && debug_path[0];
    FILE* debug_file = nullptr;
    if (debug) {                                          // create_debug_file polish.rs:230-244
        debug_file = fopen(debug_path, "wb");
        if (!debug_file) return pp_ctx_fail(ctx, PP_ERR_IO, ("unable to create \"" + std::string(debug_path) + "\"").c_str());
    }
    struct FileCloser { FILE*& f; ~FileCloser() { if (f) fclose(f); } } closer{debug_file};

    // the first SAM file starts streaming into HBM while the assembly is loaded
    if (n_sams > 0 && pp_get_parser(ctx) == 0 && n_ctx == 1) pp_tok_prefetch(ctx, sams[0]);
    char ebuf[1024];
    pp_fasta* fa = pp_fasta_load(assembly, ebuf, sizeof ebuf);
    if (!fa) return pp_ctx_fail(ctx, PP_ERR_INPUT, ebuf);
    pp_contigs contigs;
    pp_fasta_view(fa, &contigs);
    if (verbose) {
        fprintf(stderr, "Loading assembly\n");
        for (uint32_t i = 0; i < contigs.n_contigs; ++i)
            fprintf(stderr, "%s (%s bp)\n", pp_fasta_name(fa, i), fmt_thousands(contigs.off[i + 1] - contigs.off[i]).c_str());
        fprintf(stderr, "\nLoading alignments\n");
    }

    // one job per GPU; with one GPU the job is the whole assembly
    uint32_t n_shards = debug ? 1u : (uint32_t)std::max(1, std::min<int>(n_ctx, (int)contigs.n_contigs));   // the debug TSV is written from one GPU
    std::vector<ShardJob> jobs;
    int rc = PP_OK;
    pp_alignments alns;
    pp_pack* pk = nullptr;
    pp_shards* shards = nullptr;
    std::string tok_timing;
    HostCopy tok_copy;                       // the tokenised arrays back on the host (several GPUs: the sharder works there)
    bool need_host_filter = false;
    if (debug) pp_polish_set_debug(ctx, 1);
    // Pass 0 parses the SAM text in HBM (tok_kernels.cu).  Anything unusual - PP_TOK_HOST, or a data error raised by the polish
    // kernels, whose message needs read / reference names - repeats the load with the host packer (pass 1), which decides.
    for (int pass = ((n_sams > 0 && pp_get_parser(ctx) == 0) || ff) ? 0 : 1; pass < 2; ++pass) {
        if (ff && (pass == 1 || pp_get_parser(ctx) != 0)) { need_host_filter = true; break; }
        jobs.assign(n_shards, ShardJob());
        memset(&alns, 0, sizeof alns);
        bool resident = false, device_shards = false;
        rc = PP_OK;
        std::string log;
        if (pass == 0 && ff) {
            // filter (filter.rs:26-37) and the load of polish in one pass over the text: both files go to HBM once, the filter's
            // verdict becomes the ZP flag of the tokenised records (what ZP:Z:fail does after a round trip through two files)
            pp_filter_result fres;
            pp_filter_file_stats fs;
            memset(&fres, 0, sizeof fres);
            pp_fused_polish fuse;
            memset(&fuse, 0, sizeof fuse);
            fuse.fasta = fa; fuse.careful = prm->careful;
            rc = pp_filter_files_device(ctx, sams[0], sams[1], ff->out1, ff->out2, &ff->prm, &fres, &fs, &fuse);
            if (rc == PP_OK && fuse.rc == PP_TOK_HOST) rc = PP_TOK_HOST;
            if (rc == PP_TOK_HOST) { need_host_filter = true; pass = 0; break; }
            if (rc != PP_OK) { pp_fasta_free(fa); return rc; }
            static const char* nm[4] = {"fr", "rf", "ff", "rr"};
            char tmp[512];
            for (int k = 0; k < 2; ++k) {
                snprintf(tmp, sizeof tmp, "%s: %s alignments, %s pass the insert-size filter, %s fail\n", sams[k], fmt_thousands(fs.alignments[k]).c_str(),
                         fmt_thousands(fs.pass[k]).c_str(), fmt_thousands(fs.fail[k]).c_str());
                log += tmp;
            }
            snprintf(tmp, sizeof tmp, "orientation %s, insert size thresholds %u - %u\n", fres.orientation < 4 ? nm[fres.orientation] : ff->orientation.c_str(), fres.low, fres.high);
            log += tmp;
            if (n_shards > 1 || debug) rc = tok_copy.fetch(ctx, &alns);
            if (rc != PP_OK) { pp_fasta_free(fa); return rc; }
            resident = n_shards == 1;
            alns.n_aln = fuse.n_aln;
        } else if (pass == 0 && n_shards > 1) {
            // Several GPUs, no host in the middle: the host only decides which contig goes where (longest contig first onto the lightest
            // shard) and where to cut the files; the text, the records and the shards never pass through host memory as arrays.
            std::vector<uint32_t> order(contigs.n_contigs), owner(contigs.n_contigs);
            for (uint32_t i = 0; i < contigs.n_contigs; ++i) order[i] = i;
            std::stable_sort(order.begin(), order.end(), [&](uint32_t x, uint32_t y) { return contigs.off[x + 1] - contigs.off[x] > contigs.off[y + 1] - contigs.off[y]; });
            std::vector<uint64_t> load(n_shards, 0);
            for (uint32_t ci : order) {
                const uint32_t best = (uint32_t)(std::min_element(load.begin(), load.end()) - load.begin());
                owner[ci] = best;
                load[best] += contigs.off[ci + 1] - contigs.off[ci];
            }
            for (uint32_t s = 0; s < n_shards; ++s) {
                ShardJob& j = jobs[s];
                j.ctx = ctxs[s];
                j.own_local.assign(contigs.n_contigs, 0xFFFFFFFFu);
                j.own_off.assign(1, 0);
                for (uint32_t ci = 0; ci < contigs.n_contigs; ++ci) {
                    if (owner[ci] != s) continue;
                    j.own_local[ci] = (uint32_t)j.own_map.size();
                    j.own_map.push_back(ci);
                    j.own_bases.insert(j.own_bases.end(), contigs.bases + contigs.off[ci], contigs.bases + contigs.off[ci + 1]);
                    j.own_off.push_back(j.own_bases.size());
                }
                j.contigs.n_contigs = (uint32_t)j.own_map.size(); j.contigs.off = j.own_off.data(); j.contigs.bases = j.own_bases.data();
                j.contig_map = j.own_map.data();
                j.resident = true;
            }
            // every GPU reads ITS byte range of every file (cut between read groups), tokenises it, and the read groups are exchanged
            // between the GPUs (tok_kernels.cu pp_tok_exchange_finish): 1/N of the text per PCIe link
            std::vector<std::vector<uint64_t>> cuts((size_t)n_sams);
            bool ranges_ok = n_sams > 0;
            for (int i = 0; i < n_sams && ranges_ok; ++i) { ranges_ok = split_ranges(sams[i], (int)n_shards, cuts[(size_t)i]); }
            if (!ranges_ok) continue;
            std::vector<int> trc(n_shards, PP_OK);
            std::vector<std::vector<pp_tok_stats>> tst(n_shards, std::vector<pp_tok_stats>((size_t)n_sams));
            int bits = 4;
            bool host = false;
            for (int attempt = 0; attempt < 2; ++attempt) {
                auto work = [&](uint32_t s) {
                    pp_ctx* c = ctxs[s];
                    std::vector<uint64_t> off((size_t)n_sams), len((size_t)n_sams);
                    uint64_t mine = 0;
                    for (int i = 0; i < n_sams; ++i) { off[(size_t)i] = cuts[(size_t)i][s]; len[(size_t)i] = cuts[(size_t)i][s + 1] - cuts[(size_t)i][s]; mine += len[(size_t)i]; }
                    int r = pp_tok_begin(c, fa, prm->careful ? 1 : 0, bits);
                    if (r == PP_OK) r = pp_tok_expect(c, mine);
                    if (r == PP_OK) r = pp_tok_set_ranges(c, off.data(), len.data(), n_sams);
                    if (r == PP_OK) r = pp_tok_add_files(c, sams, n_sams, tst[s].data());
                    trc[s] = r;
                    if (r != PP_OK && r != PP_TOK_HOST && r != PP_TOK_NEED8) jobs[s].err = pp_last_error(c);
                };
                std::vector<std::thread> tt;
                for (uint32_t s = 1; s < n_shards; ++s) tt.emplace_back(work, s);
                work(0);
                for (auto& t : tt) t.join();
                bool need8 = false;
                host = false;
                for (uint32_t s = 0; s < n_shards; ++s) { need8 |= trc[s] == PP_TOK_NEED8; host |= trc[s] == PP_TOK_HOST; }
                if (need8 && bits == 4 && !host) { bits = 8; continue; }
                host |= need8;
                break;
            }
            if (host) continue;
            for (uint32_t s = 0; s < n_shards; ++s)
                if (trc[s] != PP_OK) { rc = pp_ctx_fail(ctx, trc[s], jobs[s].err.c_str()); pp_fasta_free(fa); return rc; }
            bool empty_file = false;
            for (int i = 0; i < n_sams; ++i) {
                uint64_t na = 0, nr = 0, nl = 0;
                float h2d = 0, dev = 0;
                for (uint32_t s = 0; s < n_shards; ++s) {
                    const pp_tok_stats& t = tst[s][(size_t)i];
                    na += t.alignments; nr += t.reads; nl += t.lines; h2d = std::max(h2d, t.h2d_ms); dev = std::max(dev, t.device_ms);
                }
                empty_file |= na == 0;                                         // "no alignments in <file>" (alignment.rs:268-270): the host path words it
                log += std::string(sams[i]) + ": " + fmt_thousands(na) + " alignments from " + fmt_thousands(nr) + " reads\n";
                char tmp[256];
                snprintf(tmp, sizeof tmp, "SAM tokeniser %s: %s lines in %u byte ranges, text to HBM %.3f ms, kernels %.3f ms (slowest GPU)\n", sams[i],
                         fmt_thousands(nl).c_str(), n_shards, h2d, dev);
                tok_timing += tmp;
            }
            if (empty_file) continue;
            {
                std::vector<const uint32_t*> lo(n_shards);
                std::vector<pp_contigs> sc(n_shards);
                for (uint32_t s = 0; s < n_shards; ++s) { lo[s] = jobs[s].own_local.data(); sc[s] = jobs[s].contigs; }
                uint64_t n_all = 0;
                const auto t0 = std::chrono::steady_clock::now();
                rc = pp_tok_exchange_finish(ctxs, (int)n_shards, owner.data(), contigs.n_contigs, lo.data(), sc.data(), &n_all);
                if (rc == PP_TOK_HOST) continue;
                if (rc != PP_OK) { pp_fasta_free(fa); return rc; }
                char tmp[160];
                snprintf(tmp, sizeof tmp, "read groups exchanged between %u GPUs and binned: %.3f ms\n", n_shards,
                         std::chrono::duration<float, std::milli>(std::chrono::steady_clock::now() - t0).count());
                tok_timing += tmp;
                alns.n_aln = n_all;
                for (uint32_t s = 0; s < n_shards; ++s) {
                    pp_alignments v;
                    if (pp_dataset_sizes(ctxs[s], &v) == PP_OK) jobs[s].alns.n_aln = v.n_aln;
                }
            }
            device_shards = true;
        } else if (pass == 0) {
            uint64_t n_aln = 0;
            rc = tokenise_files(ctx, fa, sams, n_sams, prm->careful != 0, log, tok_timing, &n_aln);
            if (rc == PP_TOK_HOST) continue;
            if (rc == PP_OK && (n_shards > 1 || debug)) rc = tok_copy.fetch(ctx, &alns);   // several GPUs: the sharder; --debug: allele strings of the TSV
            if (rc != PP_OK) { pp_fasta_free(fa); return rc; }
            resident = n_shards == 1;
            alns.n_aln = n_aln;
        } else {
            pk = pp_pack_create(fa, prm->careful);
            for (int i = 0; i < n_sams && rc == PP_OK; ++i) {
                rc = pp_pack_add_sam_file(pk, sams[i]);
                if (rc == PP_OK && verbose) {
                    uint64_t na = 0, nr = 0;
                    pp_pack_file_stats(pk, (uint32_t)i, &na, &nr);
                    fprintf(stderr, "%s: %s alignments from %s reads\n", sams[i], fmt_thousands(na).c_str(), fmt_thousands(nr).c_str());
                }
            }
            if (rc == PP_OK) rc = pp_pack_finish(pk, &alns);
            if (rc != PP_OK) {
                rc = pp_ctx_fail(ctx, rc, pp_pack_error(pk));
                pp_pack_free(pk);
                pp_fasta_free(fa);
                return rc;
            }
        }
        if (device_shards) {
            // (the jobs are set up: each context holds its shard)
        } else if (n_shards == 1) {
            jobs[0].ctx = ctx; jobs[0].contigs = contigs; jobs[0].alns = alns; jobs[0].resident = resident;
        } else {
            shards = pp_shards_build(&contigs, &alns, n_shards);
            for (uint32_t s = 0; s < n_shards; ++s) {
                jobs[s].ctx = ctxs[s];
                pp_shards_get(shards, s, &jobs[s].contigs, &jobs[s].alns, &jobs[s].contig_map, nullptr);
            }
        }
        std::vector<std::thread> th;
        for (uint32_t s = 1; s < n_shards; ++s) th.emplace_back(run_shard, &jobs[s], prm);
        run_shard(&jobs[0], prm);
        for (auto& t : th) t.join();
        bool data_error = false;
        for (auto& j : jobs) data_error |= j.rc == PP_ERR_INPUT;
        if (pass == 0 && data_error) {
            if (shards) { pp_shards_free(shards); shards = nullptr; }
            tok_timing.clear();
            if (ff) { need_host_filter = true; break; }
            continue;
        }
        if (data_error && n_shards > 1) {
            // the message names the read / reference of the offending line (alignment.rs:190-198,298-300): its index in the unsharded
            // arrays is what the packer can look up, so the failing job runs once more as one shard
            pp_shards_free(shards); shards = nullptr;
            n_shards = 1;
            jobs.assign(1, ShardJob());
            jobs[0].ctx = ctx; jobs[0].contigs = contigs; jobs[0].alns = alns; jobs[0].resident = false;
            run_shard(&jobs[0], prm);
        }
        if (verbose) fputs(log.c_str(), stderr);
        break;
    }
    if (need_host_filter) {
        // Something the fused device path leaves to the text code (a malformed line, an empty file, host parsing asked for, a data
        // error whose message needs names): the two commands one after the other, through files, exactly like the reference.
        if (shards) { pp_shards_free(shards); shards = nullptr; }
        pp_fasta_free(fa);
        if (debug) pp_polish_set_debug(ctx, 0);
        std::string t1 = ff->out1 ? ff->out1 : "", t2 = ff->out2 ? ff->out2 : "";
        char tmpl1[] = "/tmp/polypolish_filtered_1_XXXXXX", tmpl2[] = "/tmp/polypolish_filtered_2_XXXXXX";
        if (t1.empty()) { int fd = mkstemp(tmpl1); if (fd < 0) return pp_ctx_fail(ctx, PP_ERR_IO, "unable to create a temporary file for the filtered alignments"); close(fd); t1 = tmpl1; }
        if (t2.empty()) { int fd = mkstemp(tmpl2); if (fd < 0) return pp_ctx_fail(ctx, PP_ERR_IO, "unable to create a temporary file for the filtered alignments"); close(fd); t2 = tmpl2; }
        int frc = pp_filter_files(ctx, sams[0], sams[1], t1.c_str(), t2.c_str(), ff->orientation.c_str(), ff->prm.low_pct, ff->prm.high_pct, verbose);
        if (frc == PP_OK) {
            const char* fsams[2] = {t1.c_str(), t2.c_str()};
            frc = polish_files_impl(ctxs, n_ctx, assembly, fsams, 2, prm, debug_path, out_fasta, out_len, verbose, nullptr);
        }
        if (!ff->out1) unlink(t1.c_str());
        if (!ff->out2) unlink(t2.c_str());
        return frc;
    }
    uint64_t n_used = 0;
    for (uint32_t s = 0; s < n_shards && rc == PP_OK; ++s) {
        ShardJob& j = jobs[s];
        n_used += j.res.n_aln_used;
        if (j.rc == PP_OK) continue;
        rc = j.rc;
        std::string m = j.err;
        if (rc == PP_ERR_INPUT && j.res.error_aln >= 0 && n_shards == 1 && pk) {
            // re-word device-detected errors with the names the reference prints (alignment.rs:190-198,298-300)
            const char* rn = pp_pack_read_name(pk, (uint64_t)j.res.error_aln);
            if (m.rfind("query name", 0) == 0)
                m = "query name " + std::string(pp_pack_unknown_ref(pk, (uint64_t)j.res.error_aln)) + " in SAM but not in assembly";
            else if (m.rfind("CIGAR string does not", 0) == 0)
                m = "CIGAR string for read " + std::string(rn) + " does not match read sequence";
            else if (m.rfind("unexpected character", 0) == 0) {
                char cg[4096];
                pp_pack_cigar_string(pk, (uint64_t)j.res.error_aln, cg, sizeof cg);
                m = "unexpected character (other than M, =, X, I or D) in CIGAR string for read " + std::string(rn) +
                    ": \"" + cg + "\" - did you use BWA MEM to generate your alignments?";
            } else
                m += " (read " + std::string(rn) + ")";
        }
        pp_ctx_fail(ctx, rc, m.c_str());
    }
    if (debug) pp_polish_set_debug(ctx, 0 + (rc == PP_OK ? 2 : 0));      // keep the recorded data readable, stop recording
    if (rc == PP_OK && debug) {
        rc = write_debug_tsv(ctx, fa, &contigs, &alns, debug_file);
        if (rc != PP_OK && rc != PP_ERR_CUDA) rc = pp_ctx_fail(ctx, PP_ERR_IO, ("unable to write to file \"" + std::string(debug_path) + "\"").c_str());
    }
    if (rc != PP_OK) {
        if (shards) pp_shards_free(shards);
        if (pk) pp_pack_free(pk);
        pp_fasta_free(fa);
        return rc;
    }
    if (verbose) {
        fprintf(stderr, "\nFiltering for high-quality end-to-end alignments%s:\n", prm->careful ? " from reads with only one alignment" : "");
        fprintf(stderr, "  %s alignments kept\n", fmt_thousands(n_used).c_str());
        fprintf(stderr, "  %s alignments discarded\n\n", fmt_thousands(alns.n_aln - n_used).c_str());
    }

    // where each input contig's polished bases are: (job, local contig)
    std::vector<std::pair<uint32_t, uint32_t>> where(contigs.n_contigs);
    for (uint32_t s = 0; s < n_shards; ++s)
        for (uint32_t lc = 0; lc < jobs[s].contigs.n_contigs; ++lc)
            where[n_shards == 1 ? lc : jobs[s].contig_map[lc]] = {s, lc};
    // print_seq_to_stdout polish.rs:196-203, contigs in input order (polish.rs:147-152)
    std::string out;
    uint64_t total = 0;
    for (auto& j : jobs) total += j.res.out_len;
    out.reserve(total + 128 * (size_t)contigs.n_contigs);
    for (uint32_t i = 0; i < contigs.n_contigs; ++i) {
        const ShardJob& j = jobs[where[i].first];
        const uint32_t lc = where[i].second;
        out += '>';
        out += pp_fasta_name(fa, i);
        const char* d = pp_fasta_description(fa, i);
        if (d[0]) { out += ' '; out += d; }
        out += " polypolish\n";
        out.append((const char*)j.bases.data() + j.out_off[lc], j.out_off[lc + 1] - j.out_off[lc]);
        out += '\n';
        if (verbose) {
            uint64_t len = contigs.off[i + 1] - contigs.off[i];
            fprintf(stderr, "Polishing %s (%s bp):\n", pp_fasta_name(fa, i), fmt_thousands(len).c_str());
            fprintf(stderr, "  mean read depth: %.1fx\n", j.tdepth[lc] / (double)len);                       // polish.rs:208-210
            fprintf(stderr, "  %s bp %s a depth of zero (%.4f%% coverage)\n", fmt_thousands(j.zero[lc]).c_str(), j.zero[lc] == 1 ? "has" : "have",
                    100.0 * (double)(len - j.zero[lc]) / (double)len);
            fprintf(stderr, "  %s %s changed (%.4f%% of total positions)\n", fmt_thousands(j.changed[lc]).c_str(),
                    j.changed[lc] == 1 ? "position" : "positions", 100.0 * (double)j.changed[lc] / (double)len);
            const double accuracy = 100.0 - 100.0 * (double)j.changed[lc] / (double)len;
            fprintf(stderr, "  estimated pre-polishing sequence accuracy: %.4f%% (%s)\n\n", accuracy, qscore_text(accuracy).c_str());
        }
    }
    if (verbose) {
        fputs(tok_timing.c_str(), stderr);
        for (uint32_t s = 0; s < n_shards; ++s) {
            const pp_timing& t = jobs[s].res.timing;
            fprintf(stderr, "GPU job %u: %u contigs, %s alignments; device path %.3f ms (h2d + binning %.3f, goodness/k %.3f, tile %.3f, compact %.3f, d2h %.3f), %u kernels\n",
                    s, jobs[s].contigs.n_contigs, fmt_thousands(jobs[s].alns.n_aln).c_str(), t.total_ms, t.stage_ms[6], t.stage_ms[2], t.stage_ms[3],
                    t.stage_ms[4], t.stage_ms[7], t.launches);
        }
    }
    char* buf = (char*)malloc(out.size() + 1);
    if (shards) pp_shards_free(shards);
    if (pk) pp_pack_free(pk);
    pp_fasta_free(fa);
    if (!buf) return pp_ctx_fail(ctx, PP_ERR_NOMEM, "out of memory");
    memcpy(buf, out.data(), out.size());
    buf[out.size()] = 0;
    *out_fasta = buf;
    *out_len = out.size();
    return PP_OK;
}

// filter::filter (filter.rs:26-37) then polish::polish (polish.rs:26-38) on its output, as one call: same FASTA as running the two
// commands through intermediate files, which are only written when the caller names them.
extern "C" int pp_filter_polish_files(pp_ctx* ctx, const char* assembly, const char* in1, const char* in2, const char* out1, const char* out2,
                                      const char* orientation, double low, double high, const pp_polish_params* prm, char** out_fasta,
                                      uint64_t* out_len, int verbose) {
    if (!ctx) return PP_ERR_ARG;
    if (!in1 || !in2 || !orientation) return pp_ctx_fail(ctx, PP_ERR_ARG, "pp_filter_polish_files: null argument");
    {   // check_inputs filter.rs:40-53
        std::vector<std::string> a = {in1, in2};
        if (out1) a.push_back(out1);
        if (out2) a.push_back(out2);
        for (size_t i = 0; i < a.size(); ++i)
            for (size_t j = 0; j < i; ++j)
                if (a[i] == a[j]) return pp_ctx_fail(ctx, PP_ERR_INPUT, "--in1, --in2, --out1 and --out2 must all have unique values");
    }
    if (!(low > 0.0 && low < 50.0)) return pp_ctx_fail(ctx, PP_ERR_INPUT, "--low must be greater than 0 and less than 50");
    if (!(high > 50.0 && high < 100.0)) return pp_ctx_fail(ctx, PP_ERR_INPUT, "--high must be greater than 50 and less than 100");
    FusedFilter ff;
    ff.orientation = orientation;
    ff.prm.orientation = ff.orientation == "auto" ? -1 : ff.orientation == "fr" ? 0 : ff.orientation == "rf" ? 1 : ff.orientation == "ff" ? 2 : ff.orientation == "rr" ? 3 : 4;
    ff.prm.low_pct = low; ff.prm.high_pct = high; ff.prm.n_names = 0;
    ff.out1 = out1; ff.out2 = out2;
    const char* sams[2] = {in1, in2};
    return polish_files_impl(&ctx, 1, assembly, sams, 2, prm, nullptr, out_fasta, out_len, verbose, &ff);
}

extern "C" int pp_polish_files(pp_ctx* ctx, const char* assembly, const char* const* sams, int n_sams,
                               const pp_polish_params* prm, const char* debug_path, char** out_fasta,
                               uint64_t* out_len, int verbose) {
    if (!ctx) return PP_ERR_ARG;
    return polish_files_impl(&ctx, 1, assembly, sams, n_sams, prm, debug_path, out_fasta, out_len, verbose);
}

// Several GPUs of one box: contigs shard across the contexts (one host thread each); errors are reported on ctxs[0].
extern "C" int pp_polish_files_multi(pp_ctx* const* ctxs, int n_ctx, const char* assembly, const char* const* sams, int n_sams,
                                     const pp_polish_params* prm, const char* debug_path, char** out_fasta,
                                     uint64_t* out_len, int verbose) {
    if (!ctxs || n_ctx < 1 || !ctxs[0]) return PP_ERR_ARG;
    return polish_files_impl(ctxs, n_ctx, assembly, sams, n_sams, prm, debug_path, out_fasta, out_len, verbose);
}
