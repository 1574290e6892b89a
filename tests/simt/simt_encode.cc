/*
 * TEST INFRASTRUCTURE -- tests/simt/simt_encode.cc
 *
 * Compiles the product's encode DEVICE code (zxc_b200/csrc/zxc_encode.cuh and what it includes) for the CPU on top of
 * the fiber warp emulator in this directory and exposes one entry point that encodes a whole input the way
 * zxg_encode_body (zxc_gpu.cu) does: the dictionary's tables seeded once by zxc_seed_kernel's body, then every block
 * through encode_block<OPT>() unchanged on one emulated warp (lane order seeded per block), then zxc_compact_kernel
 * gathering the slots into the frame body.  Used by tests/test_encgen.py to check the encoder source byte-for-byte
 * against the reference without a GPU and under randomised lane scheduling.  Never linked into libzxc.so.
 *
 * The buffers are laid out as the product allocates them: the source with its 64 zero bytes of tail, the dictionary
 * as [dict padded][head][chain][256 code lengths], one warp's scratch of enc_layout(bs, level).total bytes and one
 * staging slot of enc_staging_stride(bs) bytes per block.  Each sits inside a guard band of a fill pattern, and every
 * staging slot is pre-filled with it, so a store outside [slot, slot + out_size) or outside the scratch is counted.
 * Guard-page mode (simt_enc_guard_pages): source, dictionary, scratch and staging are placed against PROT_NONE pages
 * instead, flush with the start (1) or the end (2) of the buffer; a load outside them ends the process with the
 * faulting buffer+offset (exit code 86).  Meant for a child process of the test that asks for it.
 */
#include <cuda_runtime.h>

#include <signal.h>
#include <stdio.h>
#include <sys/mman.h>
#include <unistd.h>

#include <vector>

/* event counters: ZXC_STAT sites run on every lane with the same value (counted on lane 0), ZXC_LANE_STAT sites count
 * one lane's own event (counted on every lane) */
extern "C" { uint64_t simt_stat[128]; }
#define ZXC_STAT(i, v) do { const uint64_t zv_ = (uint64_t)(v); if (simt::g_warp->current == 0) simt_stat[i] += zv_; } while (0)
#define ZXC_LANE_STAT(i, v) do { simt_stat[i] += (uint64_t)(v); } while (0)

#include "zxc_encode.cuh"

namespace {
const u32 PAD = 256;
const u8 FILL = 0xC3;

/* zxc_gpu.cu enc_staging_stride (a static there) */
u32 staging_stride(u32 bs) { return ((bs + 8u + 68u + 4u) + 255u) & ~255u; }

/* 0: guard bands; 1: guard pages, buffers flush with the page after the low guard; 2: flush with the high guard */
int g_guard = 0;

struct Region {
    const char* name;
    const u8* lo;
    size_t n;
};
Region g_regions[4];

/* one device-side buffer of n bytes, 16-byte aligned at mode 0 and 1, filled with FILL around the payload */
struct DevBuf {
    std::vector<u8> band;
    u8* map = nullptr;
    size_t map_len = 0;
    u8* p = nullptr;
    size_t n = 0;
    DevBuf(size_t n_, int slot, const char* name) : n(n_) {
        if (!g_guard) {
            band.assign(n + 2 * PAD + 256, FILL);
            p = (u8*)(((uintptr_t)band.data() + PAD + 255) & ~(uintptr_t)255);
        } else {
            const size_t pg = (size_t)sysconf(_SC_PAGESIZE);
            const size_t body = (n + pg - 1) / pg * pg + pg;
            map_len = body + 2 * pg;
            map = (u8*)mmap(nullptr, map_len, PROT_READ | PROT_WRITE, MAP_PRIVATE | MAP_ANONYMOUS, -1, 0);
            if (map == (u8*)MAP_FAILED) abort();
            memset(map + pg, FILL, body);
            mprotect(map, pg, PROT_NONE);
            mprotect(map + pg + body, pg, PROT_NONE);
            /* flush with the end, 16-byte aligned as the product's allocations are: n is a multiple of 16 here */
            p = g_guard == 1 ? map + pg : map + pg + body - n;
        }
        g_regions[slot] = Region{name, p, n};
    }
    ~DevBuf() {
        if (map) munmap(map, map_len);
    }
    DevBuf(const DevBuf&) = delete;
    DevBuf& operator=(const DevBuf&) = delete;
    /* bytes outside [p + lo, p + hi) that no longer hold FILL, within the band (or the mapped pages) */
    size_t stray(size_t lo, size_t hi) const {
        const u8* a = g_guard ? map + sysconf(_SC_PAGESIZE) : band.data();
        const u8* b = g_guard ? map + map_len - sysconf(_SC_PAGESIZE) : band.data() + band.size();
        size_t bad = 0;
        for (const u8* q = a; q < p + lo; q++) bad += *q != FILL;
        for (const u8* q = p + hi; q < b; q++) bad += *q != FILL;
        return bad;
    }
};

void on_segv(int, siginfo_t* si, void*) {
    const u8* a = (const u8*)si->si_addr;
    char msg[200];
    int len = snprintf(msg, sizeof msg, "simt guard: access outside the buffers at %p\n", (const void*)a);
    const Region* best = nullptr;
    ptrdiff_t best_gap = 0;
    for (const Region& r : g_regions) {
        if (!r.lo) continue;
        const ptrdiff_t d = a - r.lo, gap = d < 0 ? -d : d - (ptrdiff_t)r.n;
        if (!best || gap < best_gap) best = &r, best_gap = gap;
    }
    if (best)
        len = snprintf(msg, sizeof msg, "simt guard: access outside the buffers at %s%+td (%s holds %zu bytes)\n", best->name,
                       a - best->lo, best->name, best->n);
    if (write(2, msg, (size_t)len) < 0) _exit(87);
    _exit(86);
}

size_t up16(size_t n) { return (n + 15) & ~(size_t)15; }
}  // namespace

extern "C" void simt_enc_guard_pages(int mode) {
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

extern "C" u32 simt_enc_staging_stride(u32 bs) { return staging_stride(bs); }

/* Encodes src into n_blocks = ceil(src_size / block_size) slots of simt_enc_staging_stride(block_size) bytes at
 * `slots` (out_size[j] bytes used in slot j) and their concatenation at `body`.  dict_huf_lens: the shared literal
 * table as 256 unpacked code lengths, or NULL.  stray[0]: stores outside the slots' used bytes, stray[1]: stores outside
 * the warp's scratch.  Returns the number of rendezvous. */
extern "C" uint64_t simt_encode(const u8* src, uint64_t src_size, u32 block_size, int level, int checksum, const u8* dict,
                                u32 dict_size, const u8* dict_huf_lens, u8* slots, u32* out_size, u8* body, uint64_t seed,
                                uint64_t* stray) {
    const u32 nb = (u32)((src_size + block_size - 1) / block_size);
    const u32 sstride = staging_stride(block_size);
    const EncLayout lay = enc_layout(block_size, level);
    DevBuf in(up16(src_size + 64), 0, "src");
    memcpy(in.p, src, src_size);
    memset(in.p + src_size, 0, 64);
    const size_t dpad = ((size_t)dict_size + 16 + 255) & ~(size_t)255;
    const size_t dtot = dpad + (size_t)ENC_HASH_SIZE * 4 + (size_t)ENC_WINDOW * 2 + 256;
    const bool has_dict = dict && dict_size;
    DevBuf dct(has_dict ? dtot : 0, 1, "dict");
    DevBuf scr(lay.total, 2, "scratch");
    DevBuf stg((size_t)nb * sstride, 3, "staging");
    static u32 s_hist[256]; /* the warp's row of the kernel's __shared__ s_hist */

    EncodeParams P;
    memset(&P, 0, sizeof P);
    P.src = in.p;
    P.staging = stg.p;
    P.scratch = scr.p;
    uint64_t rendezvous = 0;
    if (has_dict) {
        memset(dct.p, 0, dtot);
        memcpy(dct.p, dict, dict_size);
        P.dict = dct.p;
        P.seed_head = (const u32*)(dct.p + dpad);
        P.seed_chain = (const unsigned short*)(dct.p + dpad + (size_t)ENC_HASH_SIZE * 4);
        if (dict_huf_lens && level >= 6) {
            u8* lens = dct.p + dpad + (size_t)ENC_HASH_SIZE * 4 + (size_t)ENC_WINDOW * 2;
            memcpy(lens, dict_huf_lens, 256);
            P.dict_huf_lens = lens;
        }
        auto seed_body = [&](unsigned) {
            zxc_seed_kernel(dct.p, dict_size, (u32)level, (u32*)P.seed_head, (unsigned short*)P.seed_chain);
        };
        rendezvous += simt::run_warp(seed_body, 0, 0, 32, seed);
    }
    P.src_size = src_size;
    P.scratch_stride = lay.total;
    P.block_size = block_size;
    P.n_blocks = nb;
    P.staging_stride = sstride;
    P.level = (u32)level;
    P.checksum = checksum ? 1u : 0u;
    P.dict_size = P.dict ? dict_size : 0;
    for (u32 j = 0; j < nb; j++) {
        const uint64_t off = (uint64_t)j * block_size;
        const u32 n = (u32)(src_size - off < block_size ? src_size - off : block_size);
        auto body_fn = [&](unsigned lane) {
            u8* dst = P.staging + (size_t)j * sstride;
            const u32 w = level >= 6 ? encode_block<true>(P, P.src + off, n, dst, P.scratch, s_hist, lane)
                                     : encode_block<false>(P, P.src + off, n, dst, P.scratch, s_hist, lane);
            __syncwarp();
            if (lane == 0) out_size[j] = w;
        };
        rendezvous += simt::run_warp(body_fn, 0, 0, ENC_CTA_THREADS, seed ? seed + j : 0);
    }
    /* stores: inside each slot only up to out_size, nothing outside the scratch */
    size_t bad_slots = stg.stray(0, (size_t)nb * sstride);
    for (u32 j = 0; j < nb; j++) {
        const u8* s = stg.p + (size_t)j * sstride;
        for (u32 k = out_size[j] < sstride ? out_size[j] : sstride; k < sstride; k++) bad_slots += s[k] != FILL;
    }
    stray[0] = bad_slots;
    stray[1] = scr.stray(0, lay.total);
    memcpy(slots, stg.p, (size_t)nb * sstride);
    /* the compaction kernel over host-side offsets, one warp */
    std::vector<unsigned long long> offs(nb ? nb : 1);
    unsigned long long acc = 0;
    for (u32 j = 0; j < nb; j++) {
        offs[j] = acc;
        acc += out_size[j];
    }
    auto compact = [&](unsigned) { zxc_compact_kernel(stg.p, sstride, offs.data(), out_size, body, nb); };
    rendezvous += simt::run_warp(compact, 0, 0, 32, seed);
    return rendezvous;
}
