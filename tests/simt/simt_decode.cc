/*
 * TEST INFRASTRUCTURE -- tests/simt/simt_decode.cc
 *
 * Compiles the product's decode DEVICE code (zxc_b200/csrc/zxc_decode.cuh and what it includes) for the CPU on top
 * of the fiber warp emulator in this directory and exposes one entry point that decodes a job table the way
 * zxc_decode_kernel does: one (emulated) warp per job, decode_job<UNITS>() unchanged.  Used by
 * tests/test_simt_decode.py to check the kernel source bit-for-bit against the reference without a GPU and under
 * randomised lane scheduling.  Never linked into libzxc.so.
 *
 * Guard-page mode (simt_guard_pages): the source, destination and dictionary buffers are placed against PROT_NONE
 * pages instead of inside 256-byte guard bands, at the bounds the product allocates (the dictionary with its 128
 * bytes of Huffman table behind it), either flush with the start of the buffer or flush with its end.  A load outside
 * them then ends the process: the SIGSEGV handler prints the faulting address as buffer+offset and exits with 86.
 * Meant for a child process of the test that asks for it.
 */
#include <cuda_runtime.h>

#include <signal.h>
#include <sys/mman.h>
#include <unistd.h>

#include <vector>

extern "C" { uint64_t simt_stat[64]; }
#define ZXC_STAT(i, v) do { const uint64_t zv_ = (uint64_t)(v); if (simt::g_warp->current == 0) simt_stat[i] += zv_; } while (0)

#include <stdio.h>
uint32_t simt_bar_issued[64], simt_bar_waited[64];
uint32_t simt_bar_base;
void simt_stage_fail(const char* what) {
    fprintf(stderr, "simt stage check failed: %s\n", what);
    abort();
}

#include "zxc_decode.cuh"
SimtStore simt_stores[64];
u32 simt_n_stores;

alignas(16) u8 smem[DECODE_SMEM_BYTES];

namespace {
const u32 PAD = 256;

/* 0: guard bands; 1: guard pages, buffers flush with the page after the low guard; 2: flush with the high guard */
int g_guard = 0;

struct Region {
    const char* name;
    const u8* lo;
    size_t n;
};
Region g_regions[3];

/* one device-side buffer of n bytes, filled with `fill` around the payload */
struct DevBuf {
    std::vector<u8> band;
    u8* map = nullptr;
    size_t map_len = 0;
    u8* p = nullptr;
    DevBuf(size_t n, u8 fill, int slot, const char* name) {
        if (!g_guard) {
            band.assign(n + 2 * PAD, fill);
            p = band.data() + PAD;
        } else {
            const size_t pg = (size_t)sysconf(_SC_PAGESIZE);
            const size_t body = (n + pg - 1) / pg * pg + pg; /* at least one readable page even for n == 0 */
            map_len = body + 2 * pg;
            map = (u8*)mmap(nullptr, map_len, PROT_READ | PROT_WRITE, MAP_PRIVATE | MAP_ANONYMOUS, -1, 0);
            if (map == (u8*)MAP_FAILED) abort();
            memset(map + pg, fill, body);
            mprotect(map, pg, PROT_NONE);
            mprotect(map + pg + body, pg, PROT_NONE);
            p = g_guard == 1 ? map + pg : map + pg + body - n;
        }
        g_regions[slot] = Region{name, p, n};
    }
    ~DevBuf() {
        if (map) munmap(map, map_len);
    }
    DevBuf(const DevBuf&) = delete;
    DevBuf& operator=(const DevBuf&) = delete;
    /* stores outside [p, p + n): the fill pattern must still be there */
    int stray_stores(size_t n, u8 fill) const {
        int bad = 0;
        const size_t span = g_guard ? 0 : PAD;
        for (size_t k = 0; k < span; k++) bad += (p[-1 - (ptrdiff_t)k] != fill) + (p[n + k] != fill);
        if (g_guard) {
            const size_t pg = (size_t)sysconf(_SC_PAGESIZE);
            for (u8* q = map + pg; q < p; q++) bad += *q != fill;
            for (u8* q = p + n; q < map + map_len - pg; q++) bad += *q != fill;
        }
        return bad;
    }
};

void on_segv(int, siginfo_t* si, void*) {
    const u8* a = (const u8*)si->si_addr;
    char msg[160];
    int len = snprintf(msg, sizeof msg, "simt guard: load outside the buffers at %p\n", (const void*)a);
    const Region* best = nullptr; /* the buffer the address is nearest to */
    ptrdiff_t best_gap = 0;
    for (const Region& r : g_regions) {
        if (!r.lo) continue;
        const ptrdiff_t d = a - r.lo, gap = d < 0 ? -d : d - (ptrdiff_t)r.n;
        if (!best || gap < best_gap) best = &r, best_gap = gap;
    }
    if (best)
        len = snprintf(msg, sizeof msg, "simt guard: load outside the buffers at %s%+td (%s holds %zu bytes)\n", best->name,
                       a - best->lo, best->name, best->n);
    if (write(2, msg, (size_t)len) < 0) _exit(87);
    _exit(86);
}
}  // namespace

extern "C" void simt_guard_pages(int mode) {
    g_guard = mode;
    if (!mode) return;
    static std::vector<u8> alt(1 << 16);
    stack_t ss;
    memset(&ss, 0, sizeof ss);
    ss.ss_sp = alt.data();
    ss.ss_size = alt.size();
    sigaltstack(&ss, nullptr);
    struct sigaction sa;
    memset(&sa, 0, sizeof sa);
    sa.sa_sigaction = on_segv;
    sa.sa_flags = SA_SIGINFO | SA_ONSTACK;
    sigaction(SIGSEGV, &sa, nullptr);
    sigaction(SIGBUS, &sa, nullptr);
}

/* the device side of one decode: source, destination and dictionary (+ its 128-byte Huffman table) as the product
 * allocates them, and the DecodeParams over them */
struct SimtDevice {
    DevBuf in, out, dct;
    std::vector<u8> scratch;
    unsigned long long counter = 0;
    DecodeParams P;
    uint64_t dst_size;
    SimtDevice(const u8* src, uint64_t src_size, uint64_t dst_size_, const zxc_b200_job_t* jobs, u32 n_jobs, i32* status,
               const u8* dict, u32 dict_size, const u8* dict_huf, u32 block_cap, u32 flags)
        : in(src_size, 0xA5, 0, "src"), out(dst_size_, 0x5A, 1, "dst"),
          dct((dict && dict_size) || dict_huf ? (size_t)dict_size + 128 : 0, 0x33, 2, "dict"), dst_size(dst_size_) {
        memcpy(in.p, src, src_size);
        if (dict && dict_size) memcpy(dct.p, dict, dict_size);
        if (dict_huf) memcpy(dct.p + dict_size, dict_huf, 128);
        const u32 stride = scr_stride(block_cap);
        scratch.assign((size_t)stride + 2 * PAD, 0x77);
        memset(&P, 0, sizeof P);
        P.src = in.p;
        P.dst = out.p;
        P.jobs = jobs;
        P.status = status;
        P.dict = (dict && dict_size) ? dct.p : nullptr;
        P.dict_huf = dict_huf ? dct.p + dict_size : nullptr;
        P.scratch = scratch.data() + PAD;
        P.counter = &counter;
        P.n_jobs = n_jobs;
        P.dict_size = dict_size;
        P.scratch_stride = stride;
        P.flags = flags;
        P.block_cap = block_cap;
    }
    /* copies the destination out; returns the stores found outside it */
    int finish(u8* dst) {
        memcpy(dst, out.p, dst_size);
        return out.stray_stores(dst_size, 0x5A);
    }
};

extern "C" uint64_t simt_decode_blocks(const u8* src, uint64_t src_size, u8* dst, uint64_t dst_size,
                                       const zxc_b200_job_t* jobs, u32 n_jobs, i32* status, const u8* dict, u32 dict_size,
                                       const u8* dict_huf, u32 block_cap, u32 flags, int units, uint64_t seed,
                                       int* oob_writes) {
    /* device buffers with a guard band either side: word loads may touch a few bytes outside, stores must not */
    SimtDevice dev(src, src_size, dst_size, jobs, n_jobs, status, dict, dict_size, dict_huf, block_cap, flags);
    const DecodeParams& P = dev.P;
    uint64_t rendezvous = 0;
    for (u32 j = 0; j < n_jobs; j++) {
        const zxc_b200_job_t job = jobs[j];
        u8* scr = P.scratch + 256; /* the lead-in zxc_decode_kernel leaves */
        u8* ring = smem;
        auto body = [&](unsigned lane) {
#if ZXC_STAGE
            simt_bar_base = smem_addr(ring) + RING_BYTES + ST_OFF_BAR;
            st_init(smem_addr(ring) + RING_BYTES, lane);
#endif
            const bool has_dict = P.dict != nullptr && P.dict_size != 0;
            const int r = units ? (has_dict ? decode_job<true, true>(P, job, scr, ring, lane) : decode_job<true, false>(P, job, scr, ring, lane))
                                : (has_dict ? decode_job<false, true>(P, job, scr, ring, lane) : decode_job<false, false>(P, job, scr, ring, lane));
            flush_wait(lane);
            __syncwarp();
            if (lane == 0) status[j] = r;
        };
        rendezvous += simt::run_warp(body, 0, 0, CTA_THREADS, seed ? seed + j : 0);
        if (simt_n_stores) simt_stage_fail("a bulk store was still in flight when the warp finished");
        for (int b = 0; b < 64; b++)
            if (simt_bar_issued[b] != simt_bar_waited[b]) simt_stage_fail("a bulk copy was still in flight when the block ended");
    }
    const int bad = dev.finish(dst);
    if (oob_writes) *oob_writes = bad;
    return rendezvous;
}

extern "C" u32 simt_scratch_stride(u32 block_cap) { return scr_stride(block_cap); }
