// batch.cpp — pp_batch_files: many whole commands (`polypolish batch`), run back to back on each of several contexts.
//
// One host thread per context takes the next job in order and runs it whole through pp_polish_files / pp_filter_polish_files on its
// own context, so a batch of isolates pays CUDA's start-up once and keeps every GPU busy.  The calling thread hands the results to
// on_done in job order.  Nothing here touches the device directly.
#include <unistd.h>
#include <chrono>
#include <condition_variable>
#include <cstdio>
#include <cstdlib>
#include <mutex>
#include <string>
#include <thread>
#include <vector>

#include "pp_ctx.cuh"
#include "pp_internal.h"

namespace {

char* dup_text(const std::string& s) {
    char* p = (char*)malloc(s.size() + 1);
    if (p) { memcpy(p, s.data(), s.size()); p[s.size()] = 0; }
    return p;
}

// The polished FASTA to `path`, created only now that the job has succeeded.  PP_OK, or PP_ERR_IO with the message on ctx.
int write_output(pp_ctx* ctx, const char* path, const char* data, uint64_t n) {
    FILE* f = fopen(path, "wb");
    if (!f) return pp_ctx_fail(ctx, PP_ERR_IO, ("unable to create \"" + std::string(path) + "\"").c_str());
    const bool ok = fwrite(data, 1, n, f) == n;
    if (fclose(f) == 0 && ok) return PP_OK;
    unlink(path);
    return pp_ctx_fail(ctx, PP_ERR_IO, ("unable to write to file \"" + std::string(path) + "\"").c_str());
}

// One job on ctx, with the context's per-job settings (report files, log sink) set for it and cleared after it.
void run_job(pp_ctx* ctx, const pp_batch_job& j, int verbose, pp_batch_result& r) {
    const auto t0 = std::chrono::steady_clock::now();
    std::string log;
    ctx->log = &log;
    pp_set_changes_file(ctx, j.changes);
    pp_set_status_file(ctx, j.status_bed);
    pp_set_vcf_file(ctx, j.vcf);
    pp_set_depth_file(ctx, j.depth_bedgraph);
    char* out = nullptr;
    uint64_t n = 0;
    int rc;
    if (!j.output || !j.output[0]) {
        rc = pp_ctx_fail(ctx, PP_ERR_ARG, "pp_batch_files: a job needs an output file");
    } else if (j.kind == PP_BATCH_POLISH) {
        rc = pp_polish_files(ctx, j.assembly, j.sams, j.n_sams, &j.params, j.debug && j.debug[0] ? j.debug : nullptr, &out, &n, verbose);
    } else if (j.kind == PP_BATCH_FILTER_POLISH) {
        rc = j.debug && j.debug[0] ? pp_ctx_fail(ctx, PP_ERR_ARG, "pp_batch_files: filter-polish takes no --debug")
                                   : pp_filter_polish_files(ctx, j.assembly, j.in1, j.in2, j.out1, j.out2, j.orientation ? j.orientation : "auto",
                                                            j.low, j.high, &j.params, &out, &n, verbose);
    } else {
        rc = pp_ctx_fail(ctx, PP_ERR_ARG, "pp_batch_files: unknown job kind");
    }
    if (rc == PP_OK) rc = write_output(ctx, j.output, out, n);
    pp_free(out);
    for (int (*clear)(pp_ctx*, const char*) : {pp_set_changes_file, pp_set_status_file, pp_set_vcf_file, pp_set_depth_file}) clear(ctx, nullptr);
    ctx->log = nullptr;
    r.rc = rc;
    r.log = dup_text(log);
    r.error = rc == PP_OK ? nullptr : dup_text(pp_last_error(ctx));
    r.wall_ms = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
}

}  // namespace

extern "C" int pp_batch_files(pp_ctx* const* ctxs, int n_ctx, const pp_batch_job* jobs, int n_jobs, pp_batch_result* results, int verbose,
                              pp_batch_done_fn on_done, void* user) {
    if (!ctxs || n_ctx < 1 || n_jobs < 0 || (n_jobs > 0 && (!jobs || !results))) return PP_ERR_ARG;
    for (int c = 0; c < n_ctx; ++c)
        if (!ctxs[c]) return PP_ERR_ARG;
    for (int i = 0; i < n_jobs; ++i) results[i] = pp_batch_result{PP_ERR_CUDA, -1, 0.0, nullptr, nullptr};

    std::mutex m;
    std::condition_variable cv;
    int next = 0, running = n_ctx;                       // the next job to take; context threads still taking jobs
    std::vector<char> done((size_t)n_jobs, 0);
    std::vector<std::pair<int, int>> stopped;             // (context, job) of each thread a CUDA error stopped
    auto worker = [&](int c) {
        for (;;) {
            int i;
            {
                std::lock_guard<std::mutex> lk(m);
                if (next >= n_jobs) break;
                i = next++;
            }
            run_job(ctxs[c], jobs[i], verbose, results[i]);
            results[i].context = c;
            std::lock_guard<std::mutex> lk(m);
            done[(size_t)i] = 1;
            cv.notify_all();
            if (results[i].rc == PP_ERR_CUDA) { stopped.push_back({c, i}); break; }
        }
        std::lock_guard<std::mutex> lk(m);
        --running;
        cv.notify_all();
    };
    std::vector<std::thread> th;
    for (int c = 0; c < n_ctx; ++c) th.emplace_back(worker, c);

    int failed = 0;
    for (int i = 0; i < n_jobs; ++i) {
        {
            std::unique_lock<std::mutex> lk(m);
            cv.wait(lk, [&] { return done[(size_t)i] || (running == 0 && i >= next); });
            if (!done[(size_t)i]) {                       // no thread is left to take it
                std::string why = "not run: every context stopped after a CUDA error (";
                for (size_t k = 0; k < stopped.size(); ++k)
                    why += (k ? "; " : "") + std::string("context ") + std::to_string(stopped[k].first) + ", GPU " +
                           std::to_string(ctxs[stopped[k].first]->device) + ", in job " + std::to_string(stopped[k].second + 1);
                results[i].error = dup_text(why + ")");
                results[i].log = dup_text("");
            }
        }
        failed += results[i].rc != PP_OK;
        if (on_done) on_done(i, &results[i], user);
    }
    for (auto& t : th) t.join();
    return failed ? PP_ERR_INPUT : PP_OK;
}
