/*
 * TEST INFRASTRUCTURE -- tests/simt/simt_sched.cc
 *
 * Direct checks of the emulator's scheduler (simt_rt.cc) on partial masks, for tests/test_encgen.py: each entry point
 * runs one small warp program and returns 0 when every lane saw what the GPU would give it.  The sched_bad_* programs
 * are undefined behaviour on the GPU; the emulator must abort on them (run them in a child process).
 */
#include <cuda_runtime.h>

/* two disjoint groups (even and odd lanes) shuffle and ballot at the same time, then the whole warp syncs */
extern "C" int sched_disjoint_groups(uint64_t seed) {
    int bad = 0;
    auto body = [&](unsigned lane) {
        const unsigned grp = (lane & 1) ? 0xAAAAAAAAu : 0x55555555u;
        const unsigned v = __shfl_sync(grp, lane * 10u, (int)(lane & 1));  /* lane 0 or lane 1 of the group */
        if (v != (lane & 1) * 10u) bad++;
        const unsigned b = __ballot_sync(grp, lane < 8);
        if (b != (grp & 0xFFu)) bad++;
        const unsigned s = __reduce_add_sync(grp, 1u);
        if (s != 16u) bad++;
        __syncwarp();
    };
    simt::run_warp(body, 0, 0, 32, seed);
    return bad;
}

/* lanes below 20 match values among themselves while the others are already at a full __syncwarp */
extern "C" int sched_masked_match(uint64_t seed) {
    int bad = 0;
    auto body = [&](unsigned lane) {
        const bool act = lane < 20;
        const unsigned am = __ballot_sync(0xFFFFFFFFu, act);
        if (act) {
            const unsigned m = __match_any_sync(am, (unsigned long long)(lane % 3));
            unsigned want = 0;
            for (unsigned k = 0; k < 20; k++)
                if (k % 3 == lane % 3) want |= 1u << k;
            if (m != want) bad++;
            if (__all_sync(am, 1) != 1 || __all_sync(am, lane != 4) != 0) bad++;
        }
        __syncwarp();
    };
    simt::run_warp(body, 0, 0, 32, seed);
    return bad;
}

/* lane 3 names a mask without itself */
extern "C" void sched_bad_mask_without_self() {
    simt::run_warp([](unsigned lane) { __syncwarp(lane == 3 ? 0x1u : 0xFFFFFFFFu); }, 0, 0, 32, 1);
}

/* lanes 16.. exit while lanes 0..15 wait at a primitive whose mask names them */
extern "C" void sched_bad_exited_lane() {
    simt::run_warp([](unsigned lane) { if (lane < 16) __syncwarp(); }, 0, 0, 32, 1);
}

/* lanes 0..15 wait at a ballot of the full warp, lanes 16.. at a __syncwarp of the full warp: no group can complete */
extern "C" void sched_bad_deadlock() {
    simt::run_warp([](unsigned lane) {
        if (lane < 16) (void)__ballot_sync(0xFFFFFFFFu, 1);
        else __syncwarp();
    }, 0, 0, 32, 1);
}
