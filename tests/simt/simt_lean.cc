/*
 * TEST INFRASTRUCTURE -- tests/simt/simt_lean.cc
 *
 * simt_decode.cc (the product's decode device code on the fiber warp emulator) plus one more entry point that decodes
 * a job table along the route zxc_gpu.cu launch_decode takes without checksum verification: every job through the
 * lean instance, decode_job<false, HAS_DICT, true>(), then every job it deferred (status D2_DEFER_STATUS) through the
 * general instance.  Built by tests/test_lean_split.py; never linked into libzxc.so.
 */
#include "simt_decode.cc"

extern "C" { uint32_t simt_lean_deferred; /* jobs the lean instance left to the general one in the last call */ }

extern "C" uint64_t simt_decode_two_stage(const u8* src, uint64_t src_size, u8* dst, uint64_t dst_size,
                                          const zxc_b200_job_t* jobs, u32 n_jobs, i32* status, const u8* dict,
                                          u32 dict_size, const u8* dict_huf, u32 block_cap, uint64_t seed, int* oob_writes) {
    /* device buffers with a guard band either side (or guard pages): word loads may touch a few bytes outside, stores
     * must not */
    SimtDevice dev(src, src_size, dst_size, jobs, n_jobs, status, dict, dict_size, dict_huf, block_cap, 0);
    const DecodeParams& P = dev.P;
    const bool has_dict = P.dict != nullptr && P.dict_size != 0;
    uint64_t rendezvous = 0;
    simt_lean_deferred = 0;
    for (int stage = 0; stage < 2; stage++) {
        const bool lean = stage == 0;
        for (u32 j = 0; j < n_jobs; j++) {
            if (!lean && status[j] != D2_DEFER_STATUS) continue;
            const zxc_b200_job_t job = jobs[j];
            u8* scr = P.scratch + 256; /* the lead-in zxc_decode_kernel leaves */
            u8* ring = smem;
            auto body = [&](unsigned lane) {
                int r;
                if (lean) r = has_dict ? decode_job<false, true, true>(P, job, scr, ring, lane) : decode_job<false, false, true>(P, job, scr, ring, lane);
                else r = has_dict ? decode_job<false, true, false>(P, job, scr, ring, lane) : decode_job<false, false, false>(P, job, scr, ring, lane);
                flush_wait(lane);
                __syncwarp();
                if (lane == 0) status[j] = r;
            };
            rendezvous += simt::run_warp(body, 0, 0, CTA_THREADS, seed ? seed + j : 0);
            if (lean && status[j] == D2_DEFER_STATUS) simt_lean_deferred++;
        }
    }
    const int bad = dev.finish(dst);
    if (oob_writes) *oob_writes = bad;
    return rendezvous;
}
