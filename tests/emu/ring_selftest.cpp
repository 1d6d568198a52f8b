// ring_selftest.cpp — drives the stage_* functions of polypolish_b200/csrc/polish_dev.cuh under the CPU emulator's strict model of
// bulk copies and mbarriers (tests/emu/cuda_emu.h) with one protocol error per scenario, so that tests/test_emu_ring.py can check
// that each error ends the run with its "ring model:" line, and that the correct protocol passes.
// TEST INFRASTRUCTURE: built and used by tests/test_emu_ring.py only.
#include "cuda_emu.h"

#include "../../polypolish_b200/csrc/polish_dev.cuh"

#include <string>

namespace {

struct Shared {
    alignas(16) unsigned char stage[2][256];
    unsigned long long bar[2];
};
alignas(16) unsigned char g_src[8][256];

// One warp, `rounds` chunks through a two-stage ring as tile_body runs them; `err` names the one thing done wrong.
void warp_body(const std::string& err, int rounds) {
    Shared& sh = *(Shared*)emu::shared_base();
    const uint32_t lane = threadIdx.x & 31;
    auto issue = [&](int c, int s) {
        const uint32_t bytes = err == "extra_tx" ? 80 : 64;
        stage_expect(&sh.bar[s], bytes);
        if (err == "second_arrival") stage_expect(&sh.bar[s], bytes);
        unsigned char* dst = sh.stage[s] + (err == "misaligned" ? 8 : 0);
        stage_copy(dst, g_src[c], 64, &sh.bar[s]);
    };
    if (lane == 0) { stage_bar_init(&sh.bar[0]); stage_bar_init(&sh.bar[1]); }
    __syncwarp();
    if (lane == 0) {
        issue(0, 0);
        if (err != "no_prologue_issue") issue(1, 1);
    }
    uint32_t parity = 0;
    for (int c = 0; c < rounds; ++c) {
        const int s = c & 1;
        if (err == "in_flight_exit" && c == rounds - 1) break;            // the last chunk is never waited for
        if (err != "early_refill") {
            stage_wait(&sh.bar[s], (parity >> s) & 1u);
            if (err != "no_flip") parity ^= 1u << s;
            if (sh.stage[s][lane] != g_src[c][lane]) {
                fprintf(stderr, "chunk %d: lane %u read %02x, not %02x\n", c, lane, sh.stage[s][lane], g_src[c][lane]);
                std::_Exit(2);
            }
        }
        __syncwarp();
        if (lane == 0 && c + 2 < rounds) issue(c + 2, s);
    }
}

}  // namespace

int main(int argc, char** argv) {
    const std::string err = argc > 1 ? argv[1] : "none";
    for (int c = 0; c < 8; ++c)
        for (int i = 0; i < 256; ++i) g_src[c][i] = (unsigned char)(c * 37 + i);
    emu::launch(1, 32, sizeof(Shared), [&] { warp_body(err, 6); });
    printf("ok\n");
    return 0;
}
