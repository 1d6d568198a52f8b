// cli_main.cpp — the `polypolish` command line, drop-in for the reference's (main.rs:23-126).
//
// Same subcommands, flag names (note the underscores), defaults and validation messages:
//   polypolish filter --in1 F --in2 F --out1 F --out2 F [--orientation auto] [--low 0.1] [--high 99.9]
//   polypolish polish [--debug F] [-i|--fraction_invalid 0.2] [-v|--fraction_valid 0.5] [-m|--max_errors 10]
//                     [-d|--min_depth 5] [--careful] <ASSEMBLY> [SAM]...
// Polished FASTA on stdout, log on stderr, "Error: <msg>" + exit 1 on user errors (misc.rs:29-33).
// Additive flags: --device N (first GPU), --gpus N (polish: contigs shard across N GPUs), --gpu-count N (filter, filter-polish: each of N
// GPUs filters a byte range of both SAM files; `filter` and `filter-polish` keep rejecting --gpus, as they always have), --quiet, --host-parse (polish: parse the
// SAM text on the host instead of on the device; same output), --changes F (polish, filter-polish: the --debug rows of the changed
// positions only), --status-bed F (polish, filter-polish: every position's --debug status as BED runs), --vcf F (polish,
// filter-polish: the polish's edits to the draft as VCF records that rebuild the polished FASTA), --depth-bedgraph F (polish,
// filter-polish: every position's --debug depth as bedGraph runs).
// Additive command: `polypolish batch MANIFEST` runs many `polish` / `filter-polish` command lines in one process (pp_batch_files).
// All compute happens in libpolypolish_b200.so on the GPU.
#include <cstdio>
#include <unistd.h>
#include <cstdlib>
#include <cstring>
#include <algorithm>
#include <chrono>
#include <fstream>
#include <map>
#include <sstream>
#include <string>
#include <vector>

#include "../../include/pp_abi.h"

static const char* BANNER =
    "  _____        _                       _  _       _     \n"
    " |  __ \\      | |                     | |(_)     | |    \n"
    " | |__) |___  | | _   _  _ __    ___  | | _  ___ | |__  \n"
    " |  ___// _ \\ | || | | || '_ \\  / _ \\ | || |/ __|| '_ \\ \n"
    " | |   | (_) || || |_| || |_) || (_) || || |\\__ \\| | | |\n"
    " |_|    \\___/ |_| \\__, || .__/  \\___/ |_||_||___/|_| |_|\n"
    "                   __/ || |                             \n"
    "                  |___/ |_|                             \n";

[[noreturn]] static void quit_with_error(const std::string& text) {   // misc.rs:29-33
    fprintf(stderr, "\nError: %s\n", text.c_str());
    exit(1);
}

static std::string usage_where;          // `batch`: "manifest line N: " while a job line is parsed, so that its errors name the line

[[noreturn]] static void usage_error(const std::string& text) {      // clap argument errors exit with 2
    fprintf(stderr, "error: %s%s\n\nFor more information, try '--help'.\n", usage_where.c_str(), text.c_str());
    exit(2);
}

static void help() {                      // `polypolish`, `polypolish -h`: the layout of clap 4's derived help (main.rs:23-42)
    fputs(BANNER, stdout);
    puts("\nshort-read polishing of long-read assemblies\ngithub.com/rrwick/Polypolish\n");
    puts("Usage: polypolish <COMMAND>\n");
    puts("Commands:\n  filter  filter paired-end alignments based on insert size\n  polish  polish a long-read assembly using short-read alignments\n"
         "  batch   run many polish / filter-polish jobs listed in a manifest, one job per GPU at a time (H100 build only)\n");
    puts("Options:\n  -h, --help     Print help\n  -V, --version  Print version");
}

static void help_filter() {               // main.rs:46-75
    puts("filter paired-end alignments based on insert size\n");
    puts("Usage: polypolish filter [OPTIONS] --in1 <IN1> --in2 <IN2> --out1 <OUT1> --out2 <OUT2>\n");
    puts("Options:");
    puts("      --in1 <IN1>                  Input SAM file - first read in pairs");
    puts("      --in2 <IN2>                  Input SAM file - first second in pairs");
    puts("      --out1 <OUT1>                Output SAM file - first read in pairs");
    puts("      --out2 <OUT2>                Output SAM file - first second in pairs");
    puts("      --orientation <ORIENTATION>  Expected pair orientation [default: auto]");
    puts("      --low <LOW>                  Low percentile threshold [default: 0.1]");
    puts("      --high <HIGH>                High percentile threshold [default: 99.9]");
    puts("  -h, --help                       Print help");
    puts("  -V, --version                    Print version");
    puts("\nH100 build, additive options: --device <N> (first GPU, default 0), --gpu-count <N> (each of N GPUs filters a byte range of both "
         "files), --quiet, --host-parse");
}

static void help_polish() {               // main.rs:77-108
    puts("polish a long-read assembly using short-read alignments\n");
    puts("Usage: polypolish polish [OPTIONS] <ASSEMBLY> [SAM]...\n");
    puts("Arguments:");
    puts("  <ASSEMBLY>  Assembly to polish (one file in FASTA format)");
    puts("  [SAM]...    Short read alignments (one or more files in SAM format)\n");
    puts("Options:");
    puts("      --debug <DEBUG>");
    puts("          Optional file to store per-base information for debugging purposes");
    puts("  -i, --fraction_invalid <FRACTION_INVALID>");
    puts("          A base must make up less than this fraction of the read depth to be considered invalid [default: 0.2]");
    puts("  -v, --fraction_valid <FRACTION_VALID>");
    puts("          A base must make up at least this fraction of the read depth to be considered valid [default: 0.5]");
    puts("  -m, --max_errors <MAX_ERRORS>");
    puts("          Ignore alignments with more than this many mismatches and indels [default: 10]");
    puts("  -d, --min_depth <MIN_DEPTH>");
    puts("          A base must occur at least this many times in the pileup to be considered valid [default: 5]");
    puts("      --careful");
    puts("          Ignore any reads with multiple alignments");
    puts("  -h, --help");
    puts("          Print help");
    puts("  -V, --version");
    puts("          Print version");
    puts("\nH100 build, additive options: --device <N> (first GPU, default 0), --gpus <N> (contigs shard over N GPUs), --quiet, --host-parse, "
         "--changes <FILE> (the --debug rows of the changed positions only), --status-bed <FILE> (every position's --debug status as BED runs), "
         "--vcf <FILE> (the edits to the draft as VCF records that rebuild the polished FASTA), "
         "--depth-bedgraph <FILE> (every position's --debug depth as bedGraph runs)");
}

// clap accepts `--name=value`, `-m5` / `-m=5` and a `--` separator (everything after it is positional): normalise those forms
// into separate tokens.  `value_shorts` = the short options that take a value.
struct Token { std::string text; bool positional; };
static std::vector<Token> normalise_args(int argc, char** argv, int first, const char* value_shorts) {
    std::vector<Token> out;
    bool rest = false;
    for (int i = first; i < argc; ++i) {
        const std::string a = argv[i];
        if (rest) { out.push_back({a, true}); continue; }
        if (a == "--") { rest = true; continue; }
        if (a.size() > 2 && a[0] == '-' && a[1] == '-') {
            const size_t eq = a.find('=');
            if (eq != std::string::npos) { out.push_back({a.substr(0, eq), false}); out.push_back({a.substr(eq + 1), true}); continue; }
        } else if (a.size() > 2 && a[0] == '-' && a[1] != '-' && strchr(value_shorts, a[1])) {
            out.push_back({a.substr(0, 2), false});
            out.push_back({a.substr(a[2] == '=' ? 3 : 2), true});
            continue;
        }
        out.push_back({a, false});
    }
    return out;
}

static double parse_f64(const char* flag, const char* s) {
    char* end = nullptr;
    double v = strtod(s, &end);
    if (!s[0] || (end && *end)) usage_error(std::string("invalid value '") + s + "' for '" + flag + "': invalid float literal");
    return v;
}
static uint32_t parse_u32(const char* flag, const char* s) {
    char* end = nullptr;
    if (s[0] == '-') usage_error(std::string("invalid value '") + s + "' for '" + flag + "': invalid digit found in string");
    unsigned long long v = strtoull(s, &end, 10);
    if (!s[0] || (end && *end) || v > 0xFFFFFFFFull) usage_error(std::string("invalid value '") + s + "' for '" + flag + "'");
    return (uint32_t)v;
}

// A one-shot process pays CUDA's start-up for every GPU the driver shows it (about a second on an 8-GPU box).  Before the first
// CUDA call the process is therefore narrowed to the GPUs it will use: CUDA_VISIBLE_DEVICES = entries [device, device + gpus) of
// the caller's own list (or of 0, 1, 2, ... when the variable is not set).  Inside the process the devices are then 0 .. gpus-1.
static bool restrict_visible_devices(int device, int gpus) {   // true: the chosen GPUs are now devices 0 .. gpus-1 of this process
    std::vector<std::string> ids;
    if (const char* cur = getenv("CUDA_VISIBLE_DEVICES")) {
        std::string s = cur, item;
        for (size_t i = 0; i <= s.size(); ++i) {
            if (i == s.size() || s[i] == ',') { if (!item.empty()) ids.push_back(item); item.clear(); }
            else item += s[i];
        }
        if ((int)ids.size() < device + gpus) return false;    // not enough entries: leave it to pp_create to report
    } else {
        for (int i = 0; i < device + gpus; ++i) ids.push_back(std::to_string(i));
    }
    std::string v;
    for (int i = device; i < device + gpus; ++i) { if (!v.empty()) v += ','; v += ids[(size_t)i]; }
    return setenv("CUDA_VISIBLE_DEVICES", v.c_str(), 1) == 0;
}

// POLYPOLISH_TIMING=1: wall-clock marks on stderr (process start-up vs the command itself)
static void mark(const char* what) {
    static const auto t0 = std::chrono::steady_clock::now();
    static const bool on = getenv("POLYPOLISH_TIMING") != nullptr;
    if (on) fprintf(stderr, "[timing] %8.1f ms  %s\n", std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count(), what);
}

// One subcommand's command line: the tokens and every option with its default (main.rs:46-108).
struct Args {
    std::vector<Token> tok;
    size_t i = 0;
    pp_polish_params prm{0.2, 0.5, 10, 5, 0};
    std::string debug, changes, status_bed, vcf, depth_bedgraph, in1, in2, out1, out2, orientation = "auto", output;
    double low = 0.1, high = 99.9;
    int device = 0, gpus = 1;
    bool quiet = false, host_parse = false;
    std::vector<std::string> pos;
    const char* value(const char* flag) {       // the value of the flag at tok[i]
        if (i + 1 >= tok.size()) usage_error(std::string("a value is required for '") + flag + "' but none was supplied");
        return tok[++i].text.c_str();
    }
};

// -i / -v / -m / -d / --careful / --changes / --status-bed / --vcf / --depth-bedgraph of `polish` and `filter-polish`
static bool polish_option(const std::string& a, Args& g) {
    if (a == "--changes") g.changes = g.value("--changes <FILE>");
    else if (a == "--status-bed") g.status_bed = g.value("--status-bed <FILE>");
    else if (a == "--vcf") g.vcf = g.value("--vcf <FILE>");
    else if (a == "--depth-bedgraph") g.depth_bedgraph = g.value("--depth-bedgraph <FILE>");
    else if (a == "-i" || a == "--fraction_invalid") g.prm.fraction_invalid = parse_f64("--fraction_invalid <FRACTION_INVALID>", g.value("--fraction_invalid"));
    else if (a == "-v" || a == "--fraction_valid") g.prm.fraction_valid = parse_f64("--fraction_valid <FRACTION_VALID>", g.value("--fraction_valid"));
    else if (a == "-m" || a == "--max_errors") g.prm.max_errors = parse_u32("--max_errors <MAX_ERRORS>", g.value("--max_errors"));
    else if (a == "-d" || a == "--min_depth") g.prm.min_depth = parse_u32("--min_depth <MIN_DEPTH>", g.value("--min_depth"));
    else if (a == "--careful") g.prm.careful = 1;
    else return false;
    return true;
}

// --in1 / --in2 / --out1 / --out2 / --orientation / --low / --high of `filter` and `filter-polish`
static bool filter_option(const std::string& a, Args& g) {
    if (a == "--in1") g.in1 = g.value("--in1 <IN1>");
    else if (a == "--in2") g.in2 = g.value("--in2 <IN2>");
    else if (a == "--out1") g.out1 = g.value("--out1 <OUT1>");
    else if (a == "--out2") g.out2 = g.value("--out2 <OUT2>");
    else if (a == "--orientation") g.orientation = g.value("--orientation <ORIENTATION>");
    else if (a == "--low") g.low = parse_f64("--low <LOW>", g.value("--low"));
    else if (a == "--high") g.high = parse_f64("--high <HIGH>", g.value("--high"));
    else return false;
    return true;
}

// --gpu-count of `filter` and `filter-polish`: GPUs [device, device + N), each filtering (and tokenising) a byte range of both files
static bool gpu_count_option(const std::string& a, Args& g) {
    if (a != "--gpu-count") return false;
    g.gpus = (int)parse_u32("--gpu-count <N>", g.value("--gpu-count <N>"));
    return true;
}

// The option loop of every subcommand: `own(a, g)` handles the subcommand's own flags (true: handled), then come --device, --gpus
// (when `gpus`), --quiet and --host-parse.  `filter` and `filter-polish` take their GPU count as --gpu-count (their own flag).  Positionals are collected when `positionals`, else they are clap's "unexpected argument".
template <class F>
static Args parse_args(int argc, char** argv, const char* value_shorts, bool positionals, bool gpus, F&& own) {
    Args g;
    g.tok = normalise_args(argc, argv, 2, value_shorts);
    for (; g.i < g.tok.size(); ++g.i) {
        const std::string& a = g.tok[g.i].text;
        if (g.tok[g.i].positional && positionals) { g.pos.push_back(a); continue; }
        if (g.tok[g.i].positional) usage_error("unexpected argument '" + a + "' found");
        if (own(a, g)) continue;
        if (a == "--device") g.device = (int)parse_u32("--device", g.value("--device"));
        else if (gpus && a == "--gpus") g.gpus = (int)parse_u32("--gpus", g.value("--gpus"));
        else if (a == "--quiet") g.quiet = true;
        else if (a == "--host-parse") g.host_parse = true;
        else if (!positionals || (a.size() > 1 && a[0] == '-' && a != "-")) usage_error("unexpected argument '" + a + "' found");
        else g.pos.push_back(a);
    }
    g.gpus = std::max(1, g.gpus);
    return g;
}

// One context per GPU [device, device + gpus) of the caller's list.
static std::vector<pp_ctx*> open_contexts(const Args& g) {
    const int base = restrict_visible_devices(g.device, g.gpus) ? 0 : g.device;
    std::vector<pp_ctx*> ctxs(g.gpus, nullptr);
    for (int d = 0; d < g.gpus; ++d)
        if (pp_create(base + d, &ctxs[d]) != PP_OK) quit_with_error("no usable H100 (sm_90) GPU: this build has no CPU fallback");
    mark("contexts created");
    if (g.host_parse) pp_set_parser(ctxs[0], 1);
    if (!g.changes.empty()) pp_set_changes_file(ctxs[0], g.changes.c_str());
    if (!g.status_bed.empty()) pp_set_status_file(ctxs[0], g.status_bed.c_str());
    if (!g.vcf.empty()) pp_set_vcf_file(ctxs[0], g.vcf.c_str());
    if (!g.depth_bedgraph.empty()) pp_set_depth_file(ctxs[0], g.depth_bedgraph.c_str());
    return ctxs;
}

// The end of every subcommand: "Error: <msg>" and exit 1 on failure, else `out` (if any) on stdout.
[[noreturn]] static void finish(const std::vector<pp_ctx*>& ctxs, int rc, const char* out, uint64_t n, bool quiet) {
    if (rc != PP_OK) { std::string m = pp_last_error(ctxs[0]); for (auto c : ctxs) pp_destroy(c); quit_with_error(m); }
    mark("command done");
    if (out) fwrite(out, 1, n, stdout);
    if (!quiet) fprintf(stderr, "Finished!\n");
    mark("output written");
    // A one-shot process has nothing left to do: the contexts, the driver's tear-down and the runtime's static destructors
    // (up to a second) are skipped - the kernel reclaims everything.  Output files first.
    if (fflush(stdout) != 0 || ferror(stdout)) quit_with_error("unable to write to stdout");
    fflush(stderr);
    _exit(0);
}

// The own options of `polish` and `filter-polish` (after -h / -V, which print and exit), and their required arguments: shared by the
// commands themselves and by the job lines of `batch`.
static bool polish_own(const std::string& a, Args& g) {
    if (a == "--debug") { g.debug = g.value("--debug <DEBUG>"); return true; }
    return polish_option(a, g);
}
static void polish_required(const Args& g) {
    if (g.pos.empty()) usage_error("the following required arguments were not provided:\n  <ASSEMBLY>");
}
static bool filter_polish_own(const std::string& a, Args& g) {
    return filter_option(a, g) || polish_option(a, g) || gpu_count_option(a, g);
}
static void filter_polish_required(const Args& g) {
    if (g.in1.empty() || g.in2.empty() || g.pos.size() != 1)
        usage_error("the following required arguments were not provided:\n  --in1 <IN1>\n  --in2 <IN2>\n  <ASSEMBLY>");
}

static void help_batch() {
    puts("run many polish / filter-polish jobs listed in a manifest in one process, one job per GPU at a time (H100 build only)\n");
    puts("Usage: polypolish batch [OPTIONS] <MANIFEST>\n");
    puts("Arguments:");
    puts("  <MANIFEST>  One job per line: `polish` or `filter-polish`, then that command's own arguments, plus --output <FILE>");
    puts("\nOptions:");
    puts("      --device <N>  First GPU [default: 0]");
    puts("      --gpus <N>    GPUs to run jobs on, one job per GPU at a time [default: 1]");
    puts("      --quiet       Print only the failed jobs");
    puts("      --host-parse  Parse the SAM text on the host (every job)");
    puts("  -h, --help        Print help");
    puts("\nManifest: blank lines and lines starting with '#' are ignored; fields are separated by spaces or tabs, so a path cannot "
         "contain whitespace; relative paths are relative to the working directory.  --output <FILE> (required) receives the polished "
         "FASTA the command would print to stdout, and is created only when the job succeeds.  --device, --gpus, --gpu-count, --quiet "
         "and --host-parse belong on the batch command line.  No two output files (FASTA, reports, --out1 / --out2) may be the same, "
         "and no job may read a file another job writes.  Log on stderr: one block per job in manifest order; exit status 1 if any job "
         "failed.");
}

// One job line of a manifest, parsed as its command would parse it.
struct BatchJob {
    int line = 0;
    std::string cmd;
    Args g;
};

// "a//b/./c/../d" relative to the working directory -> "/cwd/a/b/d": two names of one file that differ only lexically compare equal.
static std::string lexical_path(const std::string& p) {
    std::string full = p;
    if (p.empty() || p[0] != '/') {
        char cwd[4096];
        full = std::string(getcwd(cwd, sizeof cwd) ? cwd : ".") + "/" + p;
    }
    std::vector<std::string> parts;
    std::stringstream ss(full);
    for (std::string item; std::getline(ss, item, '/');) {
        if (item.empty() || item == ".") continue;
        if (item == "..") { if (!parts.empty()) parts.pop_back(); continue; }
        parts.push_back(item);
    }
    std::string out;
    for (auto& x : parts) out += "/" + x;
    return out.empty() ? "/" : out;
}

// The manifest, every line checked before any CUDA call: usage errors (exit 2) name the line.
static std::vector<BatchJob> read_manifest(const std::string& path) {
    std::ifstream in(path, std::ios::binary);
    if (!in) usage_error("unable to read the manifest \"" + path + "\"");
    std::vector<BatchJob> jobs;
    std::string text;
    for (int line = 1; std::getline(in, text); ++line) {
        if (!text.empty() && text.back() == '\r') text.pop_back();
        std::vector<std::string> f;
        std::string cur;
        for (char c : text + " ") {
            if (c == ' ' || c == '\t') { if (!cur.empty()) f.push_back(cur); cur.clear(); }
            else cur += c;
        }
        if (f.empty() || f[0][0] == '#') continue;
        usage_where = "manifest line " + std::to_string(line) + ": ";
        const bool polish = f[0] == "polish";
        if (!polish && f[0] != "filter-polish") usage_error("unrecognized command '" + f[0] + "' (a job is `polish` or `filter-polish`)");
        std::vector<char*> argv = {(char*)"polypolish"};
        for (auto& x : f) argv.push_back(&x[0]);
        BatchJob j;
        j.line = line;
        j.cmd = f[0];
        j.g = parse_args((int)argv.size(), argv.data(), "ivmd", true, polish, [polish](const std::string& a, Args& g) {
            if (a == "--output") { g.output = g.value("--output <FILE>"); return true; }
            if (a == "--device" || a == "--gpus" || a == "--gpu-count" || a == "--quiet" || a == "--host-parse")
                usage_error("'" + a + "' applies to every job: it belongs on the `polypolish batch` command line");
            if (a == "-h" || a == "--help" || a == "-V" || a == "--version") usage_error("unexpected argument '" + a + "' found");
            return polish ? polish_own(a, g) : filter_polish_own(a, g);
        });
        if (polish) polish_required(j.g);
        else filter_polish_required(j.g);
        if (j.g.output.empty()) usage_error("the following required arguments were not provided:\n  --output <FILE>");
        jobs.push_back(std::move(j));
    }
    usage_where.clear();
    if (in.bad()) usage_error("unable to read the manifest \"" + path + "\"");
    if (jobs.empty()) usage_error("the manifest \"" + path + "\" has no jobs");
    // every file a job writes is written by that job alone, and read by no job
    std::map<std::string, int> written;
    for (const BatchJob& j : jobs) {
        usage_where = "manifest line " + std::to_string(j.line) + ": ";
        const Args& g = j.g;
        for (const std::string* o : {&g.output, &g.debug, &g.changes, &g.status_bed, &g.vcf, &g.depth_bedgraph, &g.out1, &g.out2}) {
            if (o->empty()) continue;
            auto [it, fresh] = written.emplace(lexical_path(*o), j.line);
            if (!fresh) usage_error("the output file '" + *o + "' is also written by " + (it->second == j.line ? "this line" : "line " + std::to_string(it->second)));
        }
    }
    for (const BatchJob& j : jobs) {
        usage_where = "manifest line " + std::to_string(j.line) + ": ";
        std::vector<std::string> inputs = j.g.pos;
        if (!j.g.in1.empty()) inputs.push_back(j.g.in1);
        if (!j.g.in2.empty()) inputs.push_back(j.g.in2);
        for (const std::string& x : inputs) {
            auto it = written.find(lexical_path(x));
            if (it != written.end() && it->second != j.line)
                usage_error("the input file '" + x + "' is written by line " + std::to_string(it->second) + " (jobs may run in any order)");
        }
    }
    usage_where.clear();
    return jobs;
}

// What the on_done callback of `batch` prints with: one block per job, in manifest order.
struct BatchPrint {
    const std::vector<BatchJob>* jobs;
    int first_gpu;
    bool quiet;
    int failed = 0;
};

static void print_job(int i, const pp_batch_result* r, void* user) {
    BatchPrint& p = *(BatchPrint*)user;
    const BatchJob& j = (*p.jobs)[(size_t)i];
    p.failed += r->rc != PP_OK;
    if (p.quiet && r->rc == PP_OK) return;
    std::string gpu = r->context >= 0 ? "GPU " + std::to_string(p.first_gpu + r->context) : "not run";
    fprintf(stderr, "[job %d/%zu] manifest line %d: %s -> %s (%s)\n", i + 1, p.jobs->size(), j.line, j.cmd.c_str(), j.g.output.c_str(), gpu.c_str());
    if (!p.quiet && r->log) fputs(r->log, stderr);
    if (r->rc == PP_OK) fprintf(stderr, "Finished!\n");
    else fprintf(stderr, "Error: %s\n", r->error ? r->error : "unknown error");
    if (!p.quiet) fputc('\n', stderr);
    fflush(stderr);
}

[[noreturn]] static void run_batch(int argc, char** argv) {
    Args g = parse_args(argc, argv, "", true, true, [](const std::string& a, Args&) {
        if (a == "-h" || a == "--help") { help_batch(); exit(0); }
        if (a == "-V" || a == "--version") { puts("Polypolish-batch v0.6.1"); exit(0); }
        return false;
    });
    if (g.pos.empty()) usage_error("the following required arguments were not provided:\n  <MANIFEST>");
    if (g.pos.size() > 1) usage_error("unexpected argument '" + g.pos[1] + "' found");
    const std::vector<BatchJob> jobs = read_manifest(g.pos[0]);
    // every job's arguments, as pp_batch_files takes them (the strings stay in `jobs`)
    std::vector<std::vector<const char*>> sams(jobs.size());
    std::vector<pp_batch_job> bj(jobs.size());
    auto opt = [](const std::string& s) { return s.empty() ? nullptr : s.c_str(); };
    for (size_t i = 0; i < jobs.size(); ++i) {
        const Args& a = jobs[i].g;
        pp_batch_job& b = bj[i];
        memset(&b, 0, sizeof b);
        b.kind = jobs[i].cmd == "polish" ? PP_BATCH_POLISH : PP_BATCH_FILTER_POLISH;
        b.assembly = a.pos[0].c_str();
        if (b.kind == PP_BATCH_POLISH)
            for (size_t k = 1; k < a.pos.size(); ++k) sams[i].push_back(a.pos[k].c_str());
        b.sams = sams[i].data();
        b.n_sams = (int)sams[i].size();
        b.in1 = opt(a.in1); b.in2 = opt(a.in2); b.out1 = opt(a.out1); b.out2 = opt(a.out2); b.orientation = a.orientation.c_str();
        b.low = a.low; b.high = a.high; b.params = a.prm;
        b.debug = opt(a.debug); b.changes = opt(a.changes); b.status_bed = opt(a.status_bed); b.vcf = opt(a.vcf);
        b.depth_bedgraph = opt(a.depth_bedgraph);
        b.output = a.output.c_str();
    }
    std::vector<pp_ctx*> ctxs = open_contexts(g);           // (g names no report file: those are each job's own)
    for (pp_ctx* c : ctxs) pp_set_parser(c, g.host_parse ? 1 : 0);
    if (!g.quiet)
        fprintf(stderr, "Starting Polypolish batch (H100 build %s, %zu job%s, %d GPU%s)\n\n", pp_version(), jobs.size(), jobs.size() > 1 ? "s" : "",
                g.gpus, g.gpus > 1 ? "s" : "");
    BatchPrint bp{&jobs, g.device, g.quiet};
    std::vector<pp_batch_result> res(jobs.size());
    const int rc = pp_batch_files(ctxs.data(), g.gpus, bj.data(), (int)bj.size(), res.data(), g.quiet ? 0 : 1, print_job, &bp);
    if (rc == PP_ERR_ARG) quit_with_error("pp_batch_files: bad arguments");
    mark("batch done");
    if (!g.quiet) fprintf(stderr, "Batch finished: %zu job%s, %d failed\n", jobs.size(), jobs.size() > 1 ? "s" : "", bp.failed);
    fflush(stderr);
    _exit(bp.failed ? 1 : 0);                             // as finish(): the kernel reclaims the contexts
}

int main(int argc, char** argv) {
    mark("main");
    if (argc < 2) { help(); return 2; }
    std::string cmd = argv[1];
    if (cmd == "-h" || cmd == "--help") { help(); return 0; }
    if (cmd == "-V" || cmd == "--version") { puts("Polypolish v0.6.1"); return 0; }
    char* out = nullptr;
    uint64_t n = 0;
    if (cmd == "polish") {
        Args g = parse_args(argc, argv, "ivmd", true, true, [](const std::string& a, Args& g) {
            if (a == "-h" || a == "--help") { help_polish(); exit(0); }
            if (a == "-V" || a == "--version") { puts("Polypolish-polish v0.6.1"); exit(0); }
            return polish_own(a, g);
        });
        polish_required(g);
        std::vector<pp_ctx*> ctxs = open_contexts(g);
        if (!g.quiet) fprintf(stderr, "Starting Polypolish polish (H100 build %s, %d GPU%s)\n\n", pp_version(), g.gpus, g.gpus > 1 ? "s" : "");
        std::vector<const char*> sams;
        for (size_t i = 1; i < g.pos.size(); ++i) sams.push_back(g.pos[i].c_str());
        const int rc = pp_polish_files_multi(ctxs.data(), g.gpus, g.pos[0].c_str(), sams.data(), (int)sams.size(), &g.prm,
                                             g.debug.empty() ? nullptr : g.debug.c_str(), &out, &n, g.quiet ? 0 : 1);
        finish(ctxs, rc, out, n, g.quiet);
    }
    if (cmd == "filter") {
        Args g = parse_args(argc, argv, "", false, false, [](const std::string& a, Args& g) {
            if (a == "-h" || a == "--help") { help_filter(); exit(0); }
            if (a == "-V" || a == "--version") { puts("Polypolish-filter v0.6.1"); exit(0); }
            return filter_option(a, g) || gpu_count_option(a, g);
        });
        if (g.in1.empty() || g.in2.empty() || g.out1.empty() || g.out2.empty())
            usage_error("the following required arguments were not provided:\n  --in1 <IN1>\n  --in2 <IN2>\n  --out1 <OUT1>\n  --out2 <OUT2>");
        std::vector<pp_ctx*> ctxs = open_contexts(g);
        if (!g.quiet) fprintf(stderr, "Starting Polypolish filter (H100 build %s%s)\n\n", pp_version(), g.gpus > 1 ? (", " + std::to_string(g.gpus) + " GPUs").c_str() : "");
        const int rc = pp_filter_files_multi(ctxs.data(), g.gpus, g.in1.c_str(), g.in2.c_str(), g.out1.c_str(), g.out2.c_str(), g.orientation.c_str(),
                                             g.low, g.high, g.quiet ? 0 : 1);
        finish(ctxs, rc, nullptr, 0, g.quiet);
    }
    if (cmd == "filter-polish") {
        // ADDITIVE (not in the reference): `filter` and `polish` of its output as one command, no intermediate files unless named
        Args g = parse_args(argc, argv, "ivmd", true, false, [](const std::string& a, Args& g) {
            if (a == "-h" || a == "--help") {
                puts("filter paired-end alignments based on insert size, then polish the assembly with the filtered alignments (one pass, H100 build only)\n");
                puts("Usage: polypolish filter-polish [OPTIONS] --in1 <IN1> --in2 <IN2> <ASSEMBLY>\n");
                puts("Options: those of `filter` (--out1 / --out2 optional: written only when given) and of `polish` (except --debug)");
                exit(0);
            }
            return filter_polish_own(a, g);
        });
        filter_polish_required(g);
        std::vector<pp_ctx*> ctxs = open_contexts(g);
        if (!g.quiet) fprintf(stderr, "Starting Polypolish filter + polish (H100 build %s%s)\n\n", pp_version(), g.gpus > 1 ? (", " + std::to_string(g.gpus) + " GPUs").c_str() : "");
        const int rc = pp_filter_polish_files_multi(ctxs.data(), g.gpus, g.pos[0].c_str(), g.in1.c_str(), g.in2.c_str(),
                                                    g.out1.empty() ? nullptr : g.out1.c_str(), g.out2.empty() ? nullptr : g.out2.c_str(),
                                                    g.orientation.c_str(), g.low, g.high, &g.prm, &out, &n, g.quiet ? 0 : 1);
        finish(ctxs, rc, out, n, g.quiet);
    }
    if (cmd == "batch") run_batch(argc, argv);
    usage_error("unrecognized subcommand '" + cmd + "'");
}
