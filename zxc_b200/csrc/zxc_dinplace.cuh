/*
 * zxc_dinplace.cuh -- in-place frame decode in HBM (zxc_b200_decompress_inplace_device): the frame lies flush-right
 * in the caller's buffer and decodes into the same buffer from offset 0.  Stream order (zxg_decompress_inplace_device):
 *
 *   zxc_dplan_*           (zxc_dplan.cuh, unchanged) probe, SEK-guided plan, walk and job table, on the frame where
 *                         it lies in the buffer, with dst_capacity the buffer's; they only read the frame
 *   zxc_dinplace_probe    one thread: zxc_decompress_inplace's own checks (magic, file header, a plausible footer, the
 *                         margin), which come first in its order: a verdict here replaces the plan's
 *   zxc_dinplace_plan     one pass over the placed jobs: the first job of every round, and the hazard rule
 *   per round k < R:      a copy of the round's window of frame bytes into the staging area (cudaMemcpyAsync), then
 *     zxc_dinplace_round(k)   round k - 1's statuses back into the frame's status array, round k's jobs into one of
 *                             two round tables, right-aligned, and the decode counters
 *     zxc_decode_kernel       (unchanged) one launch_decode per slot over the round table, reading the staged copy
 *   zxc_dinplace_round(R) the last round's statuses
 *   zxc_dplan_check / _decide  (unchanged)
 *   zxc_dinplace_nosplit  with more than one round, a frame that needs the general split gets ZXC_ERROR_MEMORY
 *   zxc_dsplit_*          (unchanged) the general split, reading the staged copy (one round only: its DSplitArgs
 *                         source base is the staging area)
 *
 * Rounds: the frame is cut into windows [k W, (k + 1) W) of compressed bytes, W fixed on the host from the scratch, so
 * R = ceil(comp_size / W).  A job belongs to the round whose window holds its block header; round k's staged copy is
 * frame bytes [k W - 8, min(k W + W + O + 8, comp_size)), O = B + 12 the largest block the reference's encoder writes
 * at the scratch's block size B (a RAW block with its checksum).  Decode kernels see src = staging + 8 - k W, so a
 * job's frame offsets address the staged copy.
 *
 * Hazard rule (limit (a)): a job of round k < R - 1 may write only below the buffer offset where round k + 1's copy
 * starts, base + (k + 1) W - 8 (base = buffer_capacity - comp_size), and its bytes must lie inside its round's copy.
 * A job's planned span [dst_off, dst_off + dst_cap) bounds every byte it can write, so a frame that passes decodes
 * with every staged byte as it was in the intact frame; one that fails is rejected before the first buffer byte is
 * written.  DESIGN.md section 7j shows that frames the reference's encoder writes always pass.
 */
#pragma once
#include "zxc_dplan.cuh"

#define DI_THREADS 256

struct DInplaceArgs {
    DPlanArgs a;                 /* the plan's arguments: src = the frame in the buffer, dst_capacity = the buffer's */
    unsigned int* hazard;        /* set by zxc_dinplace_plan when the frame breaks the hazard rule */
    unsigned long long* rstart;  /* R + 1 entries: round k's jobs are plan jobs [rstart[k], rstart[k + 1]) */
    zxc_b200_job_t* rjobs[2];    /* two round tables of Jr entries (round k uses table k & 1) */
    i32* rstatus[2];             /* their status arrays */
    unsigned long long base;     /* buffer_capacity - comp_size: where the frame starts in the buffer */
    unsigned long long W, O;     /* window and largest block on disk */
    unsigned int R, Jr;
};

/* zxc_decompress_inplace's inplace_margin */
__device__ __forceinline__ u64 di_margin(u64 dsize, u32 bs, bool has_cs) {
    const u64 nb = (dsize + bs - 1) / bs;
    return (u64)bs + nb * (ZXF_BLOCK_HDR + (has_cs ? ZXF_BLOCK_CKS : 0)) + ZXF_BLOCK_HDR +
           (ZXF_BLOCK_HDR + nb * ZXF_SEEK_ENTRY) + ZXC_FILE_FOOTER_SIZE + ZXF_TAIL_PAD;
}

/* zxc_decompress_inplace's checks ahead of the decode (inplace_probe, then the margin), in its order */
__global__ void zxc_dinplace_probe(const DInplaceArgs I) {
    const DPlanArgs& A = I.a;
    const u8* s = A.src;
    const u64 size = A.src_size;
    *I.hazard = 0;
    long long v = 0;
    if (ld32(s) != ZXF_MAGIC) {
        v = ZXC_ERROR_BAD_MAGIC;
    } else if (s[4] != ZXF_VERSION || ld16(s + 14) != dp_hash16(ld64(s), ld64(s + 8) & 0x0000FFFFFFFFFFFFull) ||
               (s[6] & 0x0Fu) != 0 || s[5] < ZXC_BLOCK_SIZE_MIN_LOG2 || s[5] > ZXC_BLOCK_SIZE_MAX_LOG2) {
        v = ZXC_ERROR_BAD_HEADER; /* every zxf_read_file_header reject */
    } else {
        const u32 bs = 1u << s[5];
        const u64 d = ld64(s + size - ZXC_FILE_FOOTER_SIZE);
        const u64 cap = A.dst_capacity;
        if (d / bs + (d % bs != 0) > size / ZXF_BLOCK_HDR) v = ZXC_ERROR_CORRUPT_DATA; /* zxf_dsize_plausible */
        else if (d > cap || cap - d < di_margin(d, bs, (s[6] & ZXF_FLAG_CHECKSUM) != 0)) v = ZXC_ERROR_DST_TOO_SMALL;
    }
    if (v != 0) {
        *A.result = v;
        A.st->done = 1;
    }
}

/* per placed job i: the first job of each round (rounds without jobs start where the next one does), and the hazard
 * rule */
__global__ void __launch_bounds__(DI_THREADS) zxc_dinplace_plan(const DInplaceArgs I) {
    const DPlanArgs& A = I.a;
    const DPlanState* S = A.st;
    if (S->done) return;
    const u64 n_fit = S->n_fit, J = A.J, W = I.W, R = I.R;
    const u64 i = (u64)blockIdx.x * DI_THREADS + threadIdx.x;
    if (n_fit == 0) {
        if (i <= R) I.rstart[i] = 0;
        return;
    }
    if (i >= n_fit) return;
    const zxc_b200_job_t Jb = A.jobs[J - n_fit + i];
    const u64 k = Jb.src_off / W;
    const u64 k0 = i == 0 ? 0 : A.jobs[J - n_fit + i - 1].src_off / W + 1;
    for (u64 r = k0; r <= k; r++) I.rstart[r] = i;
    if (i + 1 == n_fit)
        for (u64 r = k + 1; r <= R; r++) I.rstart[r] = n_fit;
    const u64 staged_end = k * W + W + I.O; /* the round's copy reaches 8 bytes further, or to the frame's end */
    const bool outside = Jb.src_off + Jb.src_len > staged_end && staged_end + 8 < A.src_size;
    const bool overwrites = k + 1 < R && (u64)Jb.dst_off + Jb.dst_cap + 8 > I.base + (k + 1) * W;
    /* block headers are 8 bytes apart at least, so a round never holds more than Jr = W / 8 + 1 jobs; kept as a check
     * because the round table has no room beyond it */
    const bool crowded = i >= I.Jr && A.jobs[J - n_fit + i - I.Jr].src_off / W == k;
    if (outside || overwrites || crowded) *I.hazard = 1;
}

/* round k: gather round k - 1's statuses (k > 0), then place round k's jobs (k < R) right-aligned in table k & 1 and
 * preset the decode counters (dp_slot, dp_preset) as zxc_dplan_place does for the whole frame.  The hazard verdict is written here, before
 * round 0's decode. */
__global__ void __launch_bounds__(DI_THREADS) zxc_dinplace_round(const DInplaceArgs I, const u32 k) {
    const DPlanArgs& A = I.a;
    DPlanState* S = A.st;
    const u32 Jr = I.Jr;
    const u64 i = (u64)blockIdx.x * DI_THREADS + threadIdx.x;
    const bool hazard = *I.hazard != 0;
    const bool live = !S->done && !hazard; /* thread 0 below sets done only when hazard is set */
    if (k == 0 && i == 0 && !S->done && hazard) {
        *A.result = ZXC_ERROR_MEMORY;
        S->done = 1;
    }
    const u64 n_fit = live ? S->n_fit : 0;
    const u64 first = A.J - n_fit;
    if (live && k > 0) {
        const u64 a = I.rstart[k - 1], n = I.rstart[k] - a;
        if (i < n) A.status[first + a + i] = I.rstatus[(k - 1) & 1][Jr - n + i];
    }
    if (k >= I.R) return;
    u64 n = 0;
    if (live) {
        const u64 a = I.rstart[k];
        n = I.rstart[k + 1] - a;
        if (i < Jr - n) I.rstatus[k & 1][i] = 0; /* no stale deferral marks in front of the round's jobs */
        else if (i < Jr) I.rjobs[k & 1][i] = A.jobs[first + a + (i - (Jr - n))];
    }
    if (i == 0) {
        const u32 slot = live ? dp_slot(S) : DP_SLOTS;
        for (u32 t = 0; t < DP_SLOTS; t++) dp_preset(S->ctr[t], t == slot ? Jr - n : Jr);
    }
}

/* limit (b): the general split decodes every block again at its true offset, which the round schedule cannot stage */
__global__ void zxc_dinplace_nosplit(const DInplaceArgs I) {
    DPlanState* S = I.a.st;
    if (I.R > 1 && !S->done && S->split) {
        *I.a.result = ZXC_ERROR_MEMORY;
        S->done = 1;
        S->split = 0;
    }
}
