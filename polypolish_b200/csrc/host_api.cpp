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
#include <charconv>
#include <memory>
#include <string>
#include <string_view>
#include <thread>
#include <utility>
#include <vector>

#include "debug_rows.h"
#include "pp_ctx.cuh"
#include "pp_internal.h"
#include "vcf_records.h"

namespace {

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

// What a cut needs to know of one SAM line [p, p + len) (newline removed): 0 a blank line, an '@' line or an unaligned record (FLAG & 4),
// which leave the open read group open; 1 an aligned record, QNAME [p, p + qlen); 2 a line whose QNAME and FLAG do not parse (the
// tokeniser hands such a file to the host packer, so any cut will do).
static int cut_kind(const char* p, size_t len, size_t& qlen) {
    if (len && p[len - 1] == '\r') --len;
    if (len == 0 || p[0] == '@') return 0;
    const char* tab = (const char*)memchr(p, '\t', len);
    if (!tab) return 2;
    qlen = (size_t)(tab - p);
    size_t i = qlen + 1, nd = 0;
    if (i < len && p[i] == '+') ++i;
    uint64_t v = 0;
    for (; i < len && p[i] != '\t'; ++i, ++nd) {                       // FLAG as the tokeniser reads it (tok_line.h field_uint)
        const unsigned d = (unsigned)(unsigned char)p[i] - '0';
        if (d > 9) return 2;
        v = v * 10 + d;
        if (v > 0xFFFFFFFFull) return 2;
    }
    if (nd == 0 || i == len) return 2;
    return (v & 4) ? 0 : 1;
}

// Cuts a SAM file into n byte ranges for n GPUs: cut[0] = 0, cut[n] = size, every other cut a line start that splits no read group as
// the reference forms them (alignment.rs:238-264).  Blank lines, '@' lines and unaligned records leave the open group open, and a record
// with an empty QNAME joins the group of the record after it, so a cut goes right before an aligned record b only when the aligned record
// a before it has a non-empty QNAME that differs from b's (or before a line that does not parse).  Each cut moves forward from
// g * size / n to the first such place.  false: not a plain file, or a line longer than the window (the caller lets one GPU read the
// whole file instead).
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
    uint64_t b0 = 0, b1 = 0;                                            // buf holds bytes [b0, b1) of the file
    bool ok = true;
    // the line starting at `pos` (< S): its bytes [p, p + len) and where the next line starts.  false (ok = false): a read error, or a
    // line longer than the window
    auto line_at = [&](uint64_t pos, const char*& p, size_t& len, uint64_t& next) -> bool {
        for (int pass = 0; pass < 2; ++pass) {
            if (pos >= b0 && pos < b1) {
                const char* s = buf.data() + (pos - b0);
                const char* nl = (const char*)memchr(s, '\n', (size_t)(b1 - pos));
                if (nl || b1 == S) {
                    len = nl ? (size_t)(nl - s) : (size_t)(b1 - pos);
                    p = s;
                    next = pos + len + 1;
                    return true;
                }
            }
            if (pass == 1) break;
            const size_t want = (size_t)std::min<uint64_t>(W, S - pos);
            size_t got = 0;
            while (got < want) {
                const ssize_t r = pread(fd, buf.data() + got, want - got, (off_t)(pos + got));
                if (r <= 0) { ok = false; return false; }
                got += (size_t)r;
            }
            b0 = pos; b1 = pos + got;
        }
        ok = false;
        return false;
    };
    const char* p = nullptr;
    size_t len = 0, ql = 0;
    uint64_t nx = 0;
    for (int g = 1; g < n && ok; ++g) {
        uint64_t pos = std::max<uint64_t>(S / (uint64_t)n * (uint64_t)g, cut[g - 1]);
        // the first line start at or after pos (the rest of the line that holds byte pos - 1)
        if (pos > 0 && pos < S) {
            if (!line_at(pos - 1, p, len, nx)) break;
            pos = std::min(nx, S);
        }
        // ... then on to the first line a cut may go before
        bool seen = false;                                              // an aligned record since pos, QNAME qa
        std::string qa;
        while (pos < S) {
            if (!line_at(pos, p, len, nx)) break;
            const int k = cut_kind(p, len, ql);
            if (k == 2) break;
            if (k == 1) {
                if (seen && !qa.empty() && (qa.size() != ql || memcmp(qa.data(), p, ql) != 0)) break;
                seen = true;
                qa.assign(p, ql);
            }
            pos = std::min(nx, S);
        }
        if (!ok) break;
        cut[g] = std::max(pos, cut[g - 1]);
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
template <auto Free> struct Deleter { template <class T> void operator()(T* p) const { Free(p); } };
using FastaPtr = std::unique_ptr<pp_fasta, Deleter<pp_fasta_free>>;
using PackPtr = std::unique_ptr<pp_pack, Deleter<pp_pack_free>>;
using ShardsPtr = std::unique_ptr<pp_shards, Deleter<pp_shards_free>>;

// --debug / --changes / --status-bed / --depth-bedgraph: the contexts record per-position data (through pp_polish_set_debug /
// pp_polish_set_changes / pp_polish_set_status / pp_polish_set_depth) for the length of the call.  They are left in mode 2 (not
// recording, the records of this call readable) when the call succeeded, otherwise in mode 0, so that later calls neither record nor
// read stale data.
struct Recording {
    using Set = int (*)(pp_ctx*, int);
    std::vector<std::pair<Set, pp_ctx*>> on;
    bool ok = false;
    void record(Set set, pp_ctx* const* c, int n) { for (int i = 0; i < n; ++i) { on.push_back({set, c[i]}); set(c[i], 1); } }
    ~Recording() { for (auto& [set, c] : on) set(c, ok ? 2 : 0); }
};

// What one way of loading the alignments leaves for the polish: one job per GPU, whatever backs their arrays, and what to print.
struct Load {
    std::vector<ShardJob> jobs;
    pp_alignments alns{};                // all alignments; host arrays only when `pack` backs them (n_aln always)
    PackPtr pack;
    ShardsPtr shards;
    std::string log, timing;             // the reference's per-file lines (alignment.rs:266-271); timing lines
};

static void one_job(Load& ld, pp_ctx* ctx, const pp_contigs& contigs, bool resident) {
    ld.jobs.assign(1, ShardJob());
    ld.jobs[0].ctx = ctx; ld.jobs[0].contigs = contigs; ld.jobs[0].alns = ld.alns; ld.jobs[0].resident = resident;
}

static std::string alignments_line(const char* path, uint64_t n_aln, uint64_t n_reads) {
    return std::string(path) + ": " + pp::thousands(n_aln) + " alignments from " + pp::thousands(n_reads) + " reads\n";
}

// `filter` in front of `polish` in the same call (pp_filter_polish_files): the two SAM files are `sams`, this says what to filter with
struct FusedFilter {
    pp_filter_params prm;
    const char* orientation;
    const char *out1, *out2;             // filtered SAM files, or null: not written
};

// Several GPUs, no host in the middle: the host only decides which contig goes where (longest contig first onto the lightest
// shard, owner[c]) and where to cut the files (cuts[f][s], split_ranges); the text, the records and the shards never pass through
// host memory as arrays.  Each job keeps its own contigs.  PP_TOK_HOST: a file cannot be cut.
static int plan_device_shards(pp_ctx* const* ctxs, uint32_t n, const pp_contigs& contigs, const char* const* sams, int n_sams, Load& ld,
                              std::vector<uint32_t>& owner, std::vector<std::vector<uint64_t>>& cuts) {
    std::vector<uint32_t> order(contigs.n_contigs);
    owner.assign(contigs.n_contigs, 0);
    for (uint32_t i = 0; i < contigs.n_contigs; ++i) order[i] = i;
    std::stable_sort(order.begin(), order.end(), [&](uint32_t x, uint32_t y) { return contigs.off[x + 1] - contigs.off[x] > contigs.off[y + 1] - contigs.off[y]; });
    std::vector<uint64_t> load(n, 0);
    for (uint32_t ci : order) {
        const uint32_t best = (uint32_t)(std::min_element(load.begin(), load.end()) - load.begin());
        owner[ci] = best;
        load[best] += contigs.off[ci + 1] - contigs.off[ci];
    }
    ld.jobs.assign(n, ShardJob());
    for (uint32_t s = 0; s < n; ++s) {
        ShardJob& j = ld.jobs[s];
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
    cuts.assign((size_t)n_sams, {});
    for (int i = 0; i < n_sams; ++i)
        if (!split_ranges(sams[i], (int)n, cuts[(size_t)i])) return PP_TOK_HOST;
    return PP_OK;
}

static int exchange(const std::vector<uint32_t>& owner, uint32_t n_contigs, Load& ld);

// SAM files -> resident datasets through the device tokeniser (tok_kernels.cu), on the contexts of ld.jobs: job s reads bytes
// [cuts[f][s], cuts[f][s + 1]) of every file f, the whole files when there is one job.  Bases are packed 4 bits wide, 8 when a read
// needs it.  One job finishes on its own; several exchange their read groups (pp_tok_exchange_finish: 1/N of the text per PCIe link).
// PP_OK, PP_TOK_HOST (the host packer must look at the text), or an error.
static int tokenise(const pp_fasta* fa, const char* const* sams, int n_sams, int careful, const std::vector<std::vector<uint64_t>>& cuts,
                    const std::vector<uint32_t>& owner, uint32_t n_contigs, Load& ld) {
    const uint32_t n = (uint32_t)ld.jobs.size();
    std::vector<int> trc(n, PP_OK);
    std::vector<std::vector<pp_tok_stats>> tst(n, std::vector<pp_tok_stats>((size_t)n_sams));
    for (int bits = 4;; bits = 8) {
        auto work = [&](uint32_t s) {
            pp_ctx* c = ld.jobs[s].ctx;
            std::vector<uint64_t> off((size_t)n_sams), len((size_t)n_sams);
            uint64_t mine = 0;
            for (int i = 0; i < n_sams; ++i) { off[(size_t)i] = cuts[(size_t)i][s]; len[(size_t)i] = cuts[(size_t)i][s + 1] - cuts[(size_t)i][s]; mine += len[(size_t)i]; }
            int r = pp_tok_begin(c, fa, careful, bits);
            if (r == PP_OK) r = pp_tok_expect(c, mine);
            if (r == PP_OK && n > 1) r = pp_tok_set_ranges(c, off.data(), len.data(), n_sams);
            if (r == PP_OK) r = pp_tok_add_files(c, sams, n_sams, tst[s].data());
            trc[s] = r;
        };
        std::vector<std::thread> tt;
        for (uint32_t s = 1; s < n; ++s) tt.emplace_back(work, s);
        work(0);
        for (auto& t : tt) t.join();
        const bool host = std::count(trc.begin(), trc.end(), PP_TOK_HOST) > 0, need8 = std::count(trc.begin(), trc.end(), PP_TOK_NEED8) > 0;
        if (need8 && bits == 4 && !host) continue;
        if (host || need8) return PP_TOK_HOST;
        break;
    }
    for (uint32_t s = 0; s < n; ++s)
        if (trc[s] != PP_OK) return pp_ctx_fail(ld.jobs[0].ctx, trc[s], std::string(pp_last_error(ld.jobs[s].ctx)).c_str());
    uint64_t n_aln = 0;
    for (int i = 0; i < n_sams; ++i) {
        pp_tok_stats sum;
        memset(&sum, 0, sizeof sum);
        for (uint32_t s = 0; s < n; ++s) {
            const pp_tok_stats& t = tst[s][(size_t)i];
            sum.alignments += t.alignments; sum.reads += t.reads; sum.lines += t.lines; sum.launches += t.launches;
            sum.h2d_ms = std::max(sum.h2d_ms, t.h2d_ms); sum.device_ms = std::max(sum.device_ms, t.device_ms);
        }
        if (sum.alignments == 0) return PP_TOK_HOST;          // "no alignments in <file>" (alignment.rs:268-270): the host path words it
        n_aln += sum.alignments;
        ld.log += alignments_line(sams[i], sum.alignments, sum.reads);
        char tmp[256];
        snprintf(tmp, sizeof tmp, "SAM tokeniser %s: %s lines in %u byte range%s, text to HBM %.3f ms, %u kernels %.3f ms (slowest GPU)\n", sams[i],
                 pp::thousands(sum.lines).c_str(), n, n > 1 ? "s" : "", sum.h2d_ms, sum.launches, sum.device_ms);
        ld.timing += tmp;
    }
    ld.alns.n_aln = n_aln;
    if (n == 1) return pp_tok_finish(ld.jobs[0].ctx);
    return exchange(owner, n_contigs, ld);
}

// Several jobs with tokenised ranges: every read group goes to the GPUs that own its contigs (pp_tok_exchange_finish).
static int exchange(const std::vector<uint32_t>& owner, uint32_t n_contigs, Load& ld) {
    const uint32_t n = (uint32_t)ld.jobs.size();
    std::vector<pp_ctx*> ctxs(n);
    std::vector<const uint32_t*> lo(n);
    std::vector<pp_contigs> sc(n);
    for (uint32_t s = 0; s < n; ++s) { ctxs[s] = ld.jobs[s].ctx; lo[s] = ld.jobs[s].own_local.data(); sc[s] = ld.jobs[s].contigs; }
    const auto t0 = std::chrono::steady_clock::now();
    const int rc = pp_tok_exchange_finish(ctxs.data(), (int)n, owner.data(), n_contigs, lo.data(), sc.data(), &ld.alns.n_aln);
    if (rc != PP_OK) return rc;
    char tmp[160];
    snprintf(tmp, sizeof tmp, "read groups exchanged between %u GPUs and binned: %.3f ms\n", n,
             std::chrono::duration<float, std::milli>(std::chrono::steady_clock::now() - t0).count());
    ld.timing += tmp;
    for (ShardJob& j : ld.jobs) {
        pp_alignments v;
        if (pp_dataset_sizes(j.ctx, &v) == PP_OK) j.alns.n_aln = v.n_aln;
    }
    return PP_OK;
}

// The device tokeniser: one GPU reads the whole files; several each take their own contigs and a byte range of every file.
// PP_OK, PP_TOK_HOST or an error.
static int load_device(pp_ctx* const* ctxs, uint32_t n, const pp_fasta* fa, const pp_contigs& contigs, const char* const* sams, int n_sams,
                       int careful, Load& ld) {
    std::vector<uint32_t> owner;
    std::vector<std::vector<uint64_t>> cuts;
    if (n > 1) {
        const int rc = plan_device_shards(ctxs, n, contigs, sams, n_sams, ld, owner, cuts);
        if (rc != PP_OK) return rc;
        return tokenise(fa, sams, n_sams, careful, cuts, owner, contigs.n_contigs, ld);
    }
    for (int i = 0; i < n_sams; ++i) cuts.push_back({0, pp::file_size(sams[i])});
    one_job(ld, ctxs[0], contigs, true);
    const int rc = tokenise(fa, sams, n_sams, careful, cuts, owner, contigs.n_contigs, ld);
    ld.jobs[0].alns = ld.alns;
    return rc;
}

// filter (filter.rs:26-37) and the load of polish in one pass over the text: both files go to HBM once, the filter's verdict
// becomes the ZP flag of the tokenised records (what ZP:Z:fail does after a round trip through two files).  Several GPUs each filter
// and tokenise byte range g of both files (the read names meet on their owner GPU for the filter), then exchange read groups by
// contig exactly like `polish` over several GPUs.
static int load_fused(pp_ctx* const* ctxs, uint32_t n, const pp_fasta* fa, const pp_contigs& contigs, const char* const* sams, const FusedFilter& ff,
                      int careful, Load& ld) {
    pp_ctx* ctx = ctxs[0];
    pp_filter_result fres;
    pp_filter_file_stats fs;
    memset(&fres, 0, sizeof fres);
    pp_fused_polish fuse;
    memset(&fuse, 0, sizeof fuse);
    fuse.fasta = fa; fuse.careful = careful;
    std::vector<uint32_t> owner;
    std::vector<std::vector<uint64_t>> cuts;
    int rc;
    if (n == 1) {
        rc = pp_filter_files_device(ctx, sams[0], sams[1], ff.out1, ff.out2, &ff.prm, &fres, &fs, &fuse);
    } else {
        rc = plan_device_shards(ctxs, n, contigs, sams, 2, ld, owner, cuts);
        const uint64_t* c[2] = {cuts.size() == 2 ? cuts[0].data() : nullptr, cuts.size() == 2 ? cuts[1].data() : nullptr};
        if (rc == PP_OK) rc = pp_filter_files_device_multi(ctxs, (int)n, sams[0], sams[1], ff.out1, ff.out2, &ff.prm, c, &fres, &fs, &fuse);
    }
    if (rc == PP_OK && fuse.rc == PP_TOK_HOST) rc = PP_TOK_HOST;
    if (rc != PP_OK) return rc;
    static const char* nm[4] = {"fr", "rf", "ff", "rr"};
    char tmp[512];
    for (int k = 0; k < 2; ++k) {
        snprintf(tmp, sizeof tmp, "%s: %s alignments, %s pass the insert-size filter, %s fail\n", sams[k], pp::thousands(fs.alignments[k]).c_str(),
                 pp::thousands(fs.pass[k]).c_str(), pp::thousands(fs.fail[k]).c_str());
        ld.log += tmp;
    }
    snprintf(tmp, sizeof tmp, "orientation %s, insert size thresholds %u - %u\n", fres.orientation < 4 ? nm[fres.orientation] : ff.orientation, fres.low, fres.high);
    ld.log += tmp;
    ld.alns.n_aln = fuse.n_aln;
    if (n == 1) {
        one_job(ld, ctx, contigs, true);
        return PP_OK;
    }
    snprintf(tmp, sizeof tmp, "filter over %u GPUs (records to the GPU of their read name, thresholds reduced across GPUs): %.3f ms\n", n, fs.total_ms);
    ld.timing += tmp;
    return exchange(owner, contigs.n_contigs, ld);
}

// The host packer (sam_pack.cpp): the text is parsed on the host, then split into n shards by pp_shards_build.  PP_OK or an error.
static int load_host(pp_ctx* const* ctxs, uint32_t n, const pp_fasta* fa, const pp_contigs& contigs, const char* const* sams, int n_sams,
                     int careful, Load& ld) {
    ld.pack.reset(pp_pack_create(fa, careful));
    int rc = PP_OK;
    for (int i = 0; i < n_sams; ++i) {
        rc = pp_pack_add_sam_file(ld.pack.get(), sams[i]);
        if (rc != PP_OK) break;
        uint64_t na = 0, nr = 0;
        pp_pack_file_stats(ld.pack.get(), (uint32_t)i, &na, &nr);
        ld.log += alignments_line(sams[i], na, nr);
    }
    if (rc == PP_OK) rc = pp_pack_finish(ld.pack.get(), &ld.alns);
    if (rc != PP_OK) return pp_ctx_fail(ctxs[0], rc, pp_pack_error(ld.pack.get()));
    if (n == 1) {
        one_job(ld, ctxs[0], contigs, false);
        return PP_OK;
    }
    ld.shards.reset(pp_shards_build(&contigs, &ld.alns, n));
    ld.jobs.assign(n, ShardJob());
    for (uint32_t s = 0; s < n; ++s) {
        ld.jobs[s].ctx = ctxs[s];
        pp_shards_get(ld.shards.get(), s, &ld.jobs[s].contigs, &ld.jobs[s].alns, &ld.jobs[s].contig_map, nullptr);
    }
    return PP_OK;
}

// Every job on its own host thread.
static void run_jobs(std::vector<ShardJob>& jobs, const pp_polish_params* prm) {
    std::vector<std::thread> th;
    for (size_t s = 1; s < jobs.size(); ++s) th.emplace_back(run_shard, &jobs[s], prm);
    run_shard(&jobs[0], prm);
    for (auto& t : th) t.join();
}

static bool data_error(const std::vector<ShardJob>& jobs) {
    return std::any_of(jobs.begin(), jobs.end(), [](const ShardJob& j) { return j.rc == PP_ERR_INPUT; });
}

// The first failed job's error, on ctx.  A data error the device found in a one-job host run is reworded with the names the
// reference prints (alignment.rs:190-198,298-300).
static int job_error(pp_ctx* ctx, const Load& ld) {
    for (const ShardJob& j : ld.jobs) {
        if (j.rc == PP_OK) continue;
        std::string m = j.err;
        if (j.rc == PP_ERR_INPUT && j.res.error_aln >= 0 && ld.jobs.size() == 1 && ld.pack) {
            pp_pack* pk = ld.pack.get();
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
        return pp_ctx_fail(ctx, j.rc, m.c_str());
    }
    return PP_OK;
}

// print_seq_to_stdout polish.rs:196-203, contigs in input order (polish.rs:147-152), with the per-contig statistics on stderr
// (polish.rs:205-226) when verbose.
static std::string assemble(const pp_fasta* fa, const pp_contigs& contigs, const std::vector<ShardJob>& jobs, int verbose) {
    // where each input contig's polished bases are: (job, local contig)
    std::vector<std::pair<uint32_t, uint32_t>> where(contigs.n_contigs);
    for (uint32_t s = 0; s < jobs.size(); ++s)
        for (uint32_t lc = 0; lc < jobs[s].contigs.n_contigs; ++lc)
            where[jobs.size() == 1 ? lc : jobs[s].contig_map[lc]] = {s, lc};
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
            fprintf(stderr, "Polishing %s (%s bp):\n", pp_fasta_name(fa, i), pp::thousands(len).c_str());
            fprintf(stderr, "  mean read depth: %.1fx\n", j.tdepth[lc] / (double)len);                       // polish.rs:208-210
            fprintf(stderr, "  %s bp %s a depth of zero (%.4f%% coverage)\n", pp::thousands(j.zero[lc]).c_str(), j.zero[lc] == 1 ? "has" : "have",
                    100.0 * (double)(len - j.zero[lc]) / (double)len);
            fprintf(stderr, "  %s %s changed (%.4f%% of total positions)\n", pp::thousands(j.changed[lc]).c_str(),
                    j.changed[lc] == 1 ? "position" : "positions", 100.0 * (double)j.changed[lc] / (double)len);
            const double accuracy = 100.0 - 100.0 * (double)j.changed[lc] / (double)len;
            fprintf(stderr, "  estimated pre-polishing sequence accuracy: %.4f%% (%s)\n\n", accuracy, qscore_text(accuracy).c_str());
        }
    }
    return out;
}

// A global position of job j's own assembly -> (input contig, position in that contig).
static std::pair<uint32_t, uint64_t> input_position(const ShardJob& j, bool one_job, uint64_t pos) {
    const uint32_t lc = (uint32_t)(std::upper_bound(j.contigs.off, j.contigs.off + j.contigs.n_contigs + 1, pos) - j.contigs.off) - 1;
    return {one_job ? lc : j.contig_map[lc], pos - j.contigs.off[lc]};
}

// --changes / --vcf: the change rows of every job, merged in the input FASTA's contig order, then position order.  Every job reports
// the rows of its own contigs (pp_polish_changes_fetch).
struct ChangeRows {
    struct Fetched { std::vector<uint64_t> pos, off; std::vector<pp_debug_pos> rows; std::vector<uint8_t> pool; };
    struct Row { uint32_t contig; uint64_t pos; uint32_t job; uint64_t i; };
    std::vector<Fetched> got;
    std::vector<Row> order;
    const pp_debug_pos& rec(const Row& r) const { return got[r.job].rows[r.i]; }
    const uint8_t* alleles(const Row& r) const { return got[r.job].pool.data() + got[r.job].off[r.i]; }
};

// PP_OK, or an error whose message is on ctx.
static int fetch_changes(pp_ctx* ctx, const std::vector<ShardJob>& jobs, ChangeRows& cr) {
    cr.got.assign(jobs.size(), {});
    cr.order.clear();
    for (uint32_t s = 0; s < jobs.size(); ++s) {
        const ShardJob& j = jobs[s];
        ChangeRows::Fetched& g = cr.got[s];
        uint64_t n = 0, bytes = 0;
        int rc = pp_polish_changes_fetch(j.ctx, 0, nullptr, nullptr, nullptr, nullptr, 0, &n, &bytes);
        if (rc == PP_OK) {
            g.pos.resize(n); g.off.resize(n); g.rows.resize(n); g.pool.resize(bytes);
            rc = pp_polish_changes_fetch(j.ctx, n, g.pos.data(), g.rows.data(), g.off.data(), g.pool.data(), bytes, &n, &bytes);
        }
        if (rc != PP_OK) return pp_ctx_fail(ctx, rc, std::string(pp_last_error(j.ctx)).c_str());
        for (uint64_t i = 0; i < n; ++i) {
            const auto cp = input_position(j, jobs.size() == 1, g.pos[i]);
            cr.order.push_back({cp.first, cp.second, s, i});
        }
    }
    std::sort(cr.order.begin(), cr.order.end(), [](const ChangeRows::Row& a, const ChangeRows::Row& b) {
        return a.contig != b.contig ? a.contig < b.contig : a.pos < b.pos;
    });
    return PP_OK;
}

// write_debug_header / write_debug_line (polish.rs:247-266): every position of the assembly, one chunk at a time; the allele strings
// of the positions that have other alleles come from the device (k_allele_strings).  PP_ERR_CUDA: its message is on ctx; any other
// error is PP_ERR_IO, the file could not be written.
static int write_debug_tsv(pp_ctx* ctx, const pp_fasta* fa, const pp_contigs& contigs, const std::vector<ShardJob>&, const ChangeRows&,
                           FILE* f) {
    if (fputs(pp::DEBUG_HEADER, f) < 0) return PP_ERR_IO;
    const uint64_t CH = 1 << 18;
    std::vector<pp_debug_pos> recs(CH);
    std::vector<uint32_t> at;
    std::vector<uint64_t> off;
    std::vector<uint8_t> pool;
    pp::DebugRows rows;
    std::string buf;
    for (uint32_t c = 0; c < contigs.n_contigs; ++c) {
        const char* name = pp_fasta_name(fa, c);
        for (uint64_t p0 = contigs.off[c]; p0 < contigs.off[c + 1]; p0 += CH) {
            const uint64_t n = std::min<uint64_t>(CH, contigs.off[c + 1] - p0);
            int rc = pp_polish_debug_fetch(ctx, p0, n, recs.data());
            if (rc != PP_OK) return rc == PP_ERR_CUDA ? rc : PP_ERR_IO;
            at.clear();
            for (uint64_t i = 0; i < n; ++i)
                if (recs[i].n_other || recs[i].new_node != 0xFFFFFFFFu) at.push_back((uint32_t)(p0 + i));
            rc = pp_polish_debug_strings(ctx, at.data(), (uint32_t)at.size(), off, pool);
            if (rc != PP_OK) return rc == PP_ERR_CUDA ? rc : PP_ERR_IO;
            buf.clear();
            size_t k = 0;
            for (uint64_t i = 0; i < n; ++i) {
                const uint8_t* al = (k < at.size() && at[k] == p0 + i) ? pool.data() + off[k++] : nullptr;
                rows.add(buf, name, p0 + i - contigs.off[c], recs[i], al);
            }
            if (fwrite(buf.data(), 1, buf.size(), f) != buf.size()) return PP_ERR_IO;
        }
    }
    return PP_OK;
}

// --changes: the --debug header, then the --debug rows of the changed positions.  PP_ERR_IO: the file could not be written.
static int write_changes(pp_ctx*, const pp_fasta* fa, const pp_contigs&, const std::vector<ShardJob>&, const ChangeRows& cr, FILE* f) {
    std::string buf = pp::DEBUG_HEADER;
    pp::DebugRows rows;
    for (const ChangeRows::Row& r : cr.order) rows.add(buf, pp_fasta_name(fa, r.contig), r.pos, cr.rec(r), cr.alleles(r));
    return fwrite(buf.data(), 1, buf.size(), f) == buf.size() ? PP_OK : PP_ERR_IO;
}

// The allele a change row emits and its count in the row's --debug pileup column: count[0..3] for A/C/G/T, count[4] for "-", else
// the matching entry of the row's allele strings (`al`, in k_allele_strings' format; a changed row never emits the draft's own base,
// count[5]).  false: the allele is not in the pileup.
static bool emitted_allele(const pp_debug_pos& r, const uint8_t* al, std::string_view& allele, uint32_t& support) {
    const uint32_t n = pp::get_u32(al);
    const uint8_t* q = al + 4;
    for (uint32_t i = 0; i < n; ++i) q += 8 + pp::get_u32(q + 4);
    allele = r.new_node != 0xFFFFFFFFu ? std::string_view((const char*)q + 4, pp::get_u32(q)) : std::string_view((const char*)&r.new_char, 1);
    static const char* const single = "ACGT-";
    if (allele.size() == 1 && allele[0])
        if (const char* b = strchr(single, allele[0])) { support = r.count[b - single]; return true; }
    q = al + 4;
    for (uint32_t i = 0; i < n; ++i, q += 8 + pp::get_u32(q + 4))
        if (std::string_view((const char*)q + 8, pp::get_u32(q + 4)) == allele) { support = pp::get_u32(q); return true; }
    return false;
}

// --vcf: the header, then per contig in the input FASTA's order the records vcf_records.h makes of its draft and its change rows.
// PP_ERR_IO: the file could not be written; another error: its message is on ctx.
static int write_vcf(pp_ctx* ctx, const pp_fasta* fa, const pp_contigs& contigs, const std::vector<ShardJob>&, const ChangeRows& cr, FILE* f) {
    std::string buf;
    pp::vcf_header_begin(buf);
    for (uint32_t c = 0; c < contigs.n_contigs; ++c) pp::vcf_header_contig(buf, pp_fasta_name(fa, c), contigs.off[c + 1] - contigs.off[c]);
    pp::vcf_header_end(buf);
    std::vector<pp::VcfChange> ch;
    size_t k = 0;
    for (uint32_t c = 0; c < contigs.n_contigs; ++c) {
        ch.clear();
        for (; k < cr.order.size() && cr.order[k].contig == c; ++k) {
            const ChangeRows::Row& r = cr.order[k];
            pp::VcfChange v{r.pos, {}, cr.rec(r).depth, 0};
            if (!emitted_allele(cr.rec(r), cr.alleles(r), v.allele, v.support))
                return pp_ctx_fail(ctx, PP_ERR_CUDA, ("--vcf: the allele emitted at " + std::string(pp_fasta_name(fa, c)) + ":" +
                                                      std::to_string(r.pos) + " is not in its pileup").c_str());
            ch.push_back(v);
        }
        pp::vcf_records(buf, pp_fasta_name(fa, c), contigs.bases + contigs.off[c], contigs.off[c + 1] - contigs.off[c], ch.data(), ch.size());
    }
    return fwrite(buf.data(), 1, buf.size(), f) == buf.size() ? PP_OK : PP_ERR_IO;
}

// --status-bed / --depth-bedgraph: the runs of a per-position report (Fetch = pp_polish_status_fetch / pp_polish_depth_fetch) as
// "<contig>\t<start>\t<end>\t<value>" lines, the value written by Text, contigs in the input FASTA's order.  Every job reports the runs
// of its own contigs; a run never crosses a contig, so each contig's lines are its runs in order.  PP_ERR_IO: the file could not be
// written; another error: its message is on ctx.
template <class T, int (*Fetch)(pp_ctx*, uint64_t, uint64_t*, T*, uint64_t*), void (*Text)(std::string&, T)>
static int write_runs(pp_ctx* ctx, const pp_fasta* fa, const pp_contigs& contigs, const std::vector<ShardJob>& jobs, const ChangeRows&, FILE* f) {
    struct Run { uint64_t start, end; T value; };
    std::vector<std::vector<Run>> by_contig(contigs.n_contigs);
    for (const ShardJob& j : jobs) {
        uint64_t n = 0;
        int rc = Fetch(j.ctx, 0, nullptr, nullptr, &n);
        std::vector<uint64_t> start(n);
        std::vector<T> value(n);
        if (rc == PP_OK && n) rc = Fetch(j.ctx, n, start.data(), value.data(), &n);
        if (rc != PP_OK) return pp_ctx_fail(ctx, rc, std::string(pp_last_error(j.ctx)).c_str());
        const uint64_t G = j.contigs.off[j.contigs.n_contigs];
        for (uint64_t i = 0; i < n; ++i) {
            const auto cp = input_position(j, jobs.size() == 1, start[i]);
            const uint64_t end = i + 1 < n ? start[i + 1] : G;
            by_contig[cp.first].push_back({cp.second, cp.second + (end - start[i]), value[i]});
        }
    }
    std::string buf;
    char num[24];
    for (uint32_t c = 0; c < contigs.n_contigs; ++c) {
        const char* name = pp_fasta_name(fa, c);
        for (const Run& r : by_contig[c]) {          // (millions of lines for the depth runs: no snprintf)
            buf += name; buf += '\t';
            buf.append(num, std::to_chars(num, num + sizeof num, r.start).ptr); buf += '\t';
            buf.append(num, std::to_chars(num, num + sizeof num, r.end).ptr); buf += '\t';
            Text(buf, r.value); buf += '\n';
        }
    }
    return fwrite(buf.data(), 1, buf.size(), f) == buf.size() ? PP_OK : PP_ERR_IO;
}
static void status_text(std::string& buf, uint8_t status) {
    static const char* const word[6] = {"low_depth", "none", "multiple", "too_close", "kept", "changed"};
    buf += word[status < 6 ? status : 0];
}
static constexpr auto write_status_bed = write_runs<uint8_t, pp_polish_status_fetch, status_text>;
static constexpr auto write_depth_bedgraph = write_runs<uint64_t, pp_polish_depth_fetch, pp::depth_text>;

// One report file of polish_files_impl: its path ("" = not asked for), the open file and what writes it.
struct ReportFile {
    std::string path;
    int (*write)(pp_ctx*, const pp_fasta*, const pp_contigs&, const std::vector<ShardJob>&, const ChangeRows&, FILE*);
    FILE* f = nullptr;
    ~ReportFile() { if (f) fclose(f); }
};

static void print_timing(const Load& ld) {
    fputs(ld.timing.c_str(), stderr);
    for (uint32_t s = 0; s < ld.jobs.size(); ++s) {
        const ShardJob& j = ld.jobs[s];
        const pp_timing& t = j.res.timing;
        fprintf(stderr, "GPU job %u: %u contigs, %s alignments; device path %.3f ms (h2d + binning %.3f, goodness/k %.3f, tile %.3f, compact %.3f, d2h %.3f), %u kernels\n",
                s, j.contigs.n_contigs, pp::thousands(j.alns.n_aln).c_str(), t.total_ms, t.stage_ms[6], t.stage_ms[2], t.stage_ms[3],
                t.stage_ms[4], t.stage_ms[7], t.launches);
    }
}

// polish::polish (polish.rs:26-38) over one or several GPUs (contigs shard across them, SURVEY.md §8e).  With `ff` the alignments
// come from the fused device filter; PP_TOK_HOST then means that filter and polish have to run one after the other through files.
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
    // the reports in the order they are created and written: --debug, then the per-context report files
    ReportFile reports[] = {{debug_path ? debug_path : "", write_debug_tsv}, {ctx->report_path[F_CHANGES], write_changes},
                            {ctx->report_path[F_STATUS], write_status_bed}, {ctx->report_path[F_VCF], write_vcf},
                            {ctx->report_path[F_DEPTH], write_depth_bedgraph}};
    const bool debug = !reports[0].path.empty(), changes = !reports[1 + F_CHANGES].path.empty(), vcf = !reports[1 + F_VCF].path.empty();
    // create_debug_file polish.rs:230-244; the other reports are worded like it
    for (ReportFile& r : reports)
        if (!r.path.empty() && !(r.f = fopen(r.path.c_str(), "wb"))) return pp_ctx_fail(ctx, PP_ERR_IO, ("unable to create \"" + r.path + "\"").c_str());
    Recording recording;
    if (debug) recording.record(pp_polish_set_debug, &ctx, 1);
    if (changes || vcf) recording.record(pp_polish_set_changes, ctxs, n_ctx);
    if (reports[1 + F_STATUS].f) recording.record(pp_polish_set_status, ctxs, n_ctx);
    if (reports[1 + F_DEPTH].f) recording.record(pp_polish_set_depth, ctxs, n_ctx);

    // the first SAM file starts streaming into HBM while the assembly is loaded
    const bool device_parser = pp_get_parser(ctx) == 0;
    if (n_sams > 0 && device_parser && n_ctx == 1) pp_tok_prefetch(ctx, sams[0]);
    char ebuf[1024];
    const FastaPtr fa(pp_fasta_load(assembly, ebuf, sizeof ebuf));
    if (!fa) return pp_ctx_fail(ctx, PP_ERR_INPUT, ebuf);
    pp_contigs contigs;
    pp_fasta_view(fa.get(), &contigs);
    if (verbose) {
        fprintf(stderr, "Loading assembly\n");
        for (uint32_t i = 0; i < contigs.n_contigs; ++i)
            fprintf(stderr, "%s (%s bp)\n", pp_fasta_name(fa.get(), i), pp::thousands(contigs.off[i + 1] - contigs.off[i]).c_str());
        fprintf(stderr, "\nLoading alignments\n");
    }

    // one job per GPU; with one GPU the job is the whole assembly.  The debug TSV is written from one GPU.
    const uint32_t n_shards = debug ? 1u : (uint32_t)std::max(1, std::min<int>(n_ctx, (int)contigs.n_contigs));
    // The SAM text is parsed in HBM first.  Anything unusual - PP_TOK_HOST, or a data error raised by the polish kernels, whose
    // message needs read / reference names - goes to the host packer, which decides.
    Load ld;
    int rc = PP_TOK_HOST;
    if (device_parser && (ff || n_sams > 0)) {
        rc = ff ? load_fused(ctxs, n_shards, fa.get(), contigs, sams, *ff, prm->careful, ld)
                : load_device(ctxs, n_shards, fa.get(), contigs, sams, n_sams, prm->careful, ld);
        if (rc == PP_OK) run_jobs(ld.jobs, prm);
        if (rc == PP_OK && data_error(ld.jobs)) rc = PP_TOK_HOST;
        if (rc == PP_OK && verbose) fputs(ld.log.c_str(), stderr);
    }
    if (rc == PP_TOK_HOST) {
        if (ff) return PP_TOK_HOST;
        ld = Load();
        rc = load_host(ctxs, n_shards, fa.get(), contigs, sams, n_sams, prm->careful, ld);
        if (verbose) fputs(ld.log.c_str(), stderr);
        if (rc == PP_OK) run_jobs(ld.jobs, prm);
        if (rc == PP_OK && data_error(ld.jobs) && ld.jobs.size() > 1) {
            // the message names the read / reference of the offending line: its index in the unsharded arrays is what the packer can
            // look up, so the job runs once more as one shard
            ld.shards.reset();
            one_job(ld, ctx, contigs, false);
            run_shard(&ld.jobs[0], prm);
        }
    }
    if (rc == PP_OK) rc = job_error(ctx, ld);
    ChangeRows change_rows;
    for (size_t i = 0; rc == PP_OK && i < std::size(reports); ++i) {
        // the change rows once, after the debug TSV: both make their allele strings in the same device pool, and the change rows'
        // strings stay there for pp_polish_changes_fetch
        if (i == 1 + F_CHANGES && (changes || vcf)) rc = fetch_changes(ctx, ld.jobs, change_rows);
        if (rc != PP_OK || !reports[i].f) continue;
        rc = reports[i].write(ctx, fa.get(), contigs, ld.jobs, change_rows, reports[i].f);
        if (rc == PP_ERR_IO) rc = pp_ctx_fail(ctx, PP_ERR_IO, ("unable to write to file \"" + reports[i].path + "\"").c_str());
    }
    if (rc != PP_OK) return rc;
    recording.ok = true;
    if (verbose) {
        uint64_t n_used = 0;
        for (const ShardJob& j : ld.jobs) n_used += j.res.n_aln_used;
        fprintf(stderr, "\nFiltering for high-quality end-to-end alignments%s:\n", prm->careful ? " from reads with only one alignment" : "");
        fprintf(stderr, "  %s alignments kept\n", pp::thousands(n_used).c_str());
        fprintf(stderr, "  %s alignments discarded\n\n", pp::thousands(ld.alns.n_aln - n_used).c_str());
    }
    const std::string out = assemble(fa.get(), contigs, ld.jobs, verbose);
    if (verbose) print_timing(ld);
    char* buf = (char*)malloc(out.size() + 1);
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
    FusedFilter ff{{}, orientation, out1, out2};
    int rc = pp::check_filter_args(ctx, in1, in2, out1, out2, orientation, low, high, &ff.prm);
    if (rc != PP_OK) return rc;
    const char* sams[2] = {in1, in2};
    rc = polish_files_impl(&ctx, 1, assembly, sams, 2, prm, nullptr, out_fasta, out_len, verbose, &ff);
    if (rc != PP_TOK_HOST) return rc;
    // Something the fused device path leaves to the text code (a malformed line, an empty file, host parsing asked for, a data
    // error whose message needs names): the two commands one after the other, through files, exactly like the reference.
    std::string t1 = out1 ? out1 : "", t2 = out2 ? out2 : "";
    char tmpl1[] = "/tmp/polypolish_filtered_1_XXXXXX", tmpl2[] = "/tmp/polypolish_filtered_2_XXXXXX";
    if (t1.empty()) { int fd = mkstemp(tmpl1); if (fd < 0) return pp_ctx_fail(ctx, PP_ERR_IO, "unable to create a temporary file for the filtered alignments"); close(fd); t1 = tmpl1; }
    if (t2.empty()) { int fd = mkstemp(tmpl2); if (fd < 0) return pp_ctx_fail(ctx, PP_ERR_IO, "unable to create a temporary file for the filtered alignments"); close(fd); t2 = tmpl2; }
    rc = pp_filter_files(ctx, in1, in2, t1.c_str(), t2.c_str(), orientation, low, high, verbose);
    if (rc == PP_OK) {
        const char* fsams[2] = {t1.c_str(), t2.c_str()};
        rc = polish_files_impl(&ctx, 1, assembly, fsams, 2, prm, nullptr, out_fasta, out_len, verbose);
    }
    if (!out1) unlink(t1.c_str());
    if (!out2) unlink(t2.c_str());
    return rc;
}

// The same over several GPUs of one box: every GPU filters and tokenises its byte range of both files, the read names meet on their
// owner GPU for the filter, the read groups on their contigs' GPUs for the polish.  More than 32 contexts, and whatever that path does
// not settle, are the one-context call's on ctxs[0].
extern "C" int pp_filter_polish_files_multi(pp_ctx* const* ctxs, int n_ctx, const char* assembly, const char* in1, const char* in2, const char* out1,
                                            const char* out2, const char* orientation, double low, double high, const pp_polish_params* prm,
                                            char** out_fasta, uint64_t* out_len, int verbose) {
    if (!ctxs || n_ctx < 1 || !ctxs[0]) return PP_ERR_ARG;
    pp_ctx* ctx = ctxs[0];
    for (int g = 1; g < n_ctx; ++g)
        if (!ctxs[g]) return pp_ctx_fail(ctx, PP_ERR_ARG, "pp_filter_polish_files_multi: null context");
    if (n_ctx == 1 || n_ctx > 32)
        return pp_filter_polish_files(ctx, assembly, in1, in2, out1, out2, orientation, low, high, prm, out_fasta, out_len, verbose);
    if (!in1 || !in2 || !orientation) return pp_ctx_fail(ctx, PP_ERR_ARG, "pp_filter_polish_files: null argument");
    FusedFilter ff{{}, orientation, out1, out2};
    int rc = pp::check_filter_args(ctx, in1, in2, out1, out2, orientation, low, high, &ff.prm);
    if (rc != PP_OK) return rc;
    const char* sams[2] = {in1, in2};
    rc = polish_files_impl(ctxs, n_ctx, assembly, sams, 2, prm, nullptr, out_fasta, out_len, verbose, &ff);
    if (rc != PP_TOK_HOST) return rc;
    return pp_filter_polish_files(ctx, assembly, in1, in2, out1, out2, orientation, low, high, prm, out_fasta, out_len, verbose);
}

static int set_report_file(pp_ctx* ctx, int which, const char* path) {
    if (!ctx) return PP_ERR_ARG;
    ctx->report_path[which] = path ? path : "";
    return PP_OK;
}
extern "C" int pp_set_changes_file(pp_ctx* ctx, const char* path) { return set_report_file(ctx, F_CHANGES, path); }
extern "C" int pp_set_status_file(pp_ctx* ctx, const char* path) { return set_report_file(ctx, F_STATUS, path); }
extern "C" int pp_set_vcf_file(pp_ctx* ctx, const char* path) { return set_report_file(ctx, F_VCF, path); }
extern "C" int pp_set_depth_file(pp_ctx* ctx, const char* path) { return set_report_file(ctx, F_DEPTH, path); }

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
