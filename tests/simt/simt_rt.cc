/* TEST INFRASTRUCTURE -- tests/simt/simt_rt.cc: fiber scheduler of the emulated warp (x86-64 System V only). */
#include "cuda_runtime.h"

extern "C" void simt_switch(void** save_sp, void* load_sp);
asm(R"(
.text
.globl simt_switch
.type simt_switch,@function
simt_switch:
    pushq %rbp
    pushq %rbx
    pushq %r12
    pushq %r13
    pushq %r14
    pushq %r15
    movq %rsp, (%rdi)
    movq %rsi, %rsp
    popq %r15
    popq %r14
    popq %r13
    popq %r12
    popq %rbx
    popq %rbp
    ret
.size simt_switch,.-simt_switch
)");

namespace simt {

thread_local Warp* g_warp = nullptr;
static const size_t STACK_BYTES = 256 * 1024;

uint64_t rendezvous(int op, uint64_t val, unsigned arg, unsigned mask) {
    Warp* w = g_warp;
    LaneCtx& me = w->lane[w->current];
    if (!(mask >> w->current & 1u)) {
        fprintf(stderr, "simt: lane %d calls op %d with mask %08x, which does not name it\n", w->current, op, mask);
        abort();
    }
    me.op = op;
    me.val = val;
    me.arg = arg;
    me.mask = mask;
    simt_switch(&me.sp, w->sched_sp);
    return me.result;
}

static void fiber_main() {
    Warp* w = g_warp;
    const int l = w->current;
    w->body((unsigned)l);
    w->lane[l].done = true;
    w->lane[l].op = OP_EXIT;
    simt_switch(&w->lane[l].sp, w->sched_sp);
    fprintf(stderr, "simt: resumed a finished lane\n");
    abort();
}

static uint64_t next_rand(uint64_t& s) {
    s ^= s << 13;
    s ^= s >> 7;
    s ^= s << 17;
    return s;
}

/* results of one completed group: every lane of mask m is parked at op */
static void complete(Warp* w, int op, unsigned m) {
    uint64_t red = 0;
    switch (op) {
        case OP_BALLOT:
        case OP_OR:
            for (int l = 0; l < 32; l++)
                if (m >> l & 1) red |= (op == OP_BALLOT) ? (uint64_t)(w->lane[l].val != 0) << l : w->lane[l].val;
            break;
        case OP_MAX:
            for (int l = 0; l < 32; l++)
                if ((m >> l & 1) && (uint32_t)w->lane[l].val > red) red = (uint32_t)w->lane[l].val;
            break;
        case OP_MIN:
            red = 0xFFFFFFFFull;
            for (int l = 0; l < 32; l++)
                if ((m >> l & 1) && (uint32_t)w->lane[l].val < red) red = (uint32_t)w->lane[l].val;
            break;
        case OP_ADD:
            for (int l = 0; l < 32; l++)
                if (m >> l & 1) red = (uint32_t)(red + w->lane[l].val);
            break;
        default: break;
    }
    for (int l = 0; l < 32; l++) {
        if (!(m >> l & 1)) continue;
        LaneCtx& c = w->lane[l];
        switch (op) {
            case OP_SYNC: c.result = 0; break;
            case OP_BALLOT: case OP_OR: case OP_MAX: case OP_MIN: case OP_ADD: c.result = red; break;
            case OP_MATCH: {
                uint64_t mm = 0;
                for (int k = 0; k < 32; k++)
                    if ((m >> k & 1) && w->lane[k].val == c.val) mm |= 1ull << k;
                c.result = mm;
                break;
            }
            /* a source lane outside the mask (undefined on the GPU) reads the value it last passed */
            case OP_SHFL_IDX: c.result = w->lane[c.arg & 31].val; break;
            case OP_SHFL_UP: c.result = (unsigned)l >= c.arg ? w->lane[l - (int)c.arg].val : c.val; break;
            case OP_SHFL_DOWN: c.result = (unsigned)l + c.arg < 32 ? w->lane[l + (int)c.arg].val : c.val; break;
            case OP_SHFL_XOR: c.result = w->lane[(l ^ (int)c.arg) & 31].val; break;
            default: fprintf(stderr, "simt: bad op %d\n", op); abort();
        }
    }
}

uint64_t run_warp(const std::function<void(unsigned)>& body, unsigned first_tid, unsigned block_idx, unsigned block_dim,
                  uint64_t seed) {
    Warp* w = new Warp();
    Warp* outer = g_warp;
    g_warp = w;
    w->body = body;
    w->rng = seed ? seed * 0x9E3779B97F4A7C15ull + 1 : 0;
    w->n_rendezvous = 0;
    for (int l = 0; l < 32; l++) {
        LaneCtx& c = w->lane[l];
        c.tid = dim3{first_tid + (unsigned)l, 0, 0};
        c.bid = dim3{block_idx, 0, 0};
        c.bdim = dim3{block_dim, 1, 1};
        c.done = false;
        c.op = OP_NONE;
        c.stack = aligned_alloc(64, STACK_BYTES);
        uintptr_t top = ((uintptr_t)c.stack + STACK_BYTES) & ~(uintptr_t)15;
        void** sp = (void**)top;
        *--sp = nullptr;                 /* fake return address of fiber_main */
        *--sp = (void*)&fiber_main;      /* `ret` target of the first switch */
        for (int r = 0; r < 6; r++) *--sp = nullptr;
        c.sp = sp;
    }
    int order[32];
    unsigned run = 0xFFFFFFFFu; /* lanes to resume this round: all at first, then the members of completed groups */
    for (;;) {
        int n = 0;
        for (int l = 0; l < 32; l++)
            if (run >> l & 1) order[n++] = l;
        if (w->rng)
            for (int i = n - 1; i > 0; i--) {
                const int j = (int)(next_rand(w->rng) % (uint64_t)(i + 1));
                const int t = order[i];
                order[i] = order[j];
                order[j] = t;
            }
        for (int i = 0; i < n; i++) {
            w->current = order[i];
            w->lane[order[i]].op = OP_NONE;
            simt_switch(&w->sched_sp, w->lane[order[i]].sp);
        }
        /* every lane is now parked at a rendezvous or has exited */
        unsigned parked = 0, exited = 0;
        for (int l = 0; l < 32; l++) {
            if (w->lane[l].done) exited |= 1u << l;
            else parked |= 1u << l;
        }
        if (!parked) break;
        /* complete every group whose lanes all wait at the same op with the same mask; two such groups are disjoint */
        run = 0;
        for (int l = 0; l < 32; l++) {
            if (!(parked >> l & 1) || (run >> l & 1)) continue;
            const int op = w->lane[l].op;
            const unsigned m = w->lane[l].mask;
            if (m & exited) {
                fprintf(stderr, "simt: lanes %08x named in mask %08x of op %d (lane %d) have exited\n", m & exited, m, op, l);
                abort();
            }
            bool ready = true;
            for (int k = 0; k < 32; k++)
                if ((m >> k & 1) && (w->lane[k].op != op || w->lane[k].mask != m)) ready = false;
            if (!ready) continue;
            complete(w, op, m);
            run |= m;
            w->n_rendezvous++;
        }
        if (!run) {
            for (int l = 0; l < 32; l++)
                if (parked >> l & 1)
                    fprintf(stderr, "simt: lane %d waits at op %d with mask %08x\n", l, w->lane[l].op, w->lane[l].mask);
            fprintf(stderr, "simt: deadlock: no group of parked lanes can complete (a lane of a mask waits at another op or mask)\n");
            abort();
        }
    }
    const uint64_t n_rv = w->n_rendezvous;
    for (int l = 0; l < 32; l++) free(w->lane[l].stack);
    g_warp = outer;
    delete w;
    return n_rv;
}

}  // namespace simt
