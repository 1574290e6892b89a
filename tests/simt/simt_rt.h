/* TEST INFRASTRUCTURE -- tests/simt/simt_rt.h: 32 fibers = one emulated warp (see cuda_runtime.h here). */
#pragma once
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>

#include <functional>

namespace simt {

enum { OP_NONE = 0, OP_SYNC, OP_BALLOT, OP_MAX, OP_MIN, OP_ADD, OP_OR, OP_MATCH, OP_SHFL_IDX, OP_SHFL_UP, OP_SHFL_DOWN, OP_SHFL_XOR, OP_EXIT };

struct LaneCtx {
    dim3 tid, bid, bdim;
    void* sp;          /* saved stack pointer of the parked fiber */
    void* stack;
    int op;            /* pending rendezvous */
    uint64_t val;
    unsigned arg;
    unsigned mask;     /* the lanes that take part in it */
    uint64_t result;
    bool done;
};

struct Warp {
    LaneCtx lane[32];
    void* sched_sp;
    int current;
    uint64_t rng;
    uint64_t n_rendezvous;
    std::function<void(unsigned)> body;
};

extern thread_local Warp* g_warp;

static inline LaneCtx& cur() { return g_warp->lane[g_warp->current]; }
uint64_t rendezvous(int op, uint64_t val, unsigned arg, unsigned mask);

/* runs body(lane) on 32 fibers to completion; block/threads describe threadIdx for lane l as first_tid + l.
 * seed != 0: lanes are resumed in a random order between rendezvous; seed == 0: lane order.  Returns the number of
 * rendezvous groups completed.  Aborts (a finding: undefined behaviour on the GPU) when a lane names a mask without
 * itself, a mask names a lane that has exited, or the parked lanes can complete no group. */
uint64_t run_warp(const std::function<void(unsigned)>& body, unsigned first_tid, unsigned block_idx, unsigned block_dim,
                  uint64_t seed);

}  // namespace simt
