/*
 * zxc_gpu.cu -- the single CUDA translation unit behind libzxc: kernels (included .cuh files) and
 * the thin extern "C" shim the host C code calls (zxc_gpu.h) -- device bring-up, contexts, staging
 * copies, launches.
 *
 * Decode launches (launch_decode below):
 *   zxc_decode_kernel   (zxc_decode.cuh)  one warp per block, any block size / section encoding: every launch by
 *                       default (instances: sequence-centric or output-centric body, with / without dictionary);
 *                       without checksum verification its lean instance runs first and the general one decodes
 *                       what the lean one deferred (GHI blocks, Huffman sections)
 * Encode: zxc_encode.cuh (levels 1-5), zxc_encode_opt.cuh (levels 6-7); the frame of a device-to-device compress
 * is assembled by zxc_assemble.cuh, and a batch of them is encoded and assembled by zxc_cbatch.cuh.
 * Dictionary training: zxc_train.cuh (zxg_train_* at the end of this file).
 */
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <pthread.h>

#include "zxc_error.h"
#include "zxc_gpu.h"

#include "zxc_decode.cuh"
#include "zxc_encode.cuh"
#include "zxc_assemble.cuh"
#include "zxc_c2host.cuh"
#include "zxc_dbatch.cuh"
#include "zxc_cbatch.cuh"
#include "zxc_dplan.cuh"
#include "zxc_dinplace.cuh"
#include "zxc_dseek.cuh"
#include "zxc_dindex.cuh"
#include "zxc_blocks.cuh"
#include "zxc_pstream_device.cuh"
#include "zxc_train.cuh"

/* ========================================================================= */
/* host side: device bring-up, contexts, copies, launches                    */
/* ========================================================================= */
static pthread_once_t g_once = PTHREAD_ONCE_INIT;
static int g_init_rc = ZXC_B200_ERROR_NO_DEVICE;
static int g_sm_count = 0;
static unsigned long long g_launches = 0;
static pthread_mutex_t g_pool_mu = PTHREAD_MUTEX_INITIALIZER;

#define PIN_CHUNK ((size_t)32 << 20)

/* ------------------------------------------------------------------------- */
/* Host copy pool.  Pageable caller buffers are staged through pinned bounce  */
/* buffers; one thread's memcpy (~10 GB/s) is far below a PCIe Gen5 link, so   */
/* copies are cut into slices that a few persistent threads claim.  There is   */
/* one pool per device, created on first use, its threads bound to the CPUs of  */
/* the device's NUMA node (/sys/bus/pci/devices/<bdf>/numa_node), which is also */
/* where the bounce buffers are placed: on the 8-GPU hosts GPUs 0-3 hang off    */
/* node 0 and 4-7 off node 1, and unplaced staging memory made the 8-rank       */
/* host-to-host figure of round 1 fall below the 4-rank one.                    */
/* ------------------------------------------------------------------------- */
#include <sched.h>
#include <sys/mman.h>
#include <sys/syscall.h>
#include <time.h>
#include <unistd.h>

#define POOL_MAX_DEV 16
#define POOL_MAX_THREADS 32
#define POOL_SLICE ((size_t)512 << 10)

extern "C" void zxh_stream_copy(void* dst, const void* src, size_t n); /* zxc_hostcopy.c */

struct copy_pool {
    pthread_mutex_t job_mu; /* one job at a time */
    pthread_mutex_t mu;
    pthread_cond_t cv_go, cv_done;
    pthread_t th[POOL_MAX_THREADS];
    int n_threads, started;
    int numa_node; /* -1 unknown */
    cpu_set_t cpus;
    int have_cpus;
    /* current job */
    u8* d;
    const u8* s;
    size_t bytes;
    size_t next; /* next slice offset (atomic) */
    unsigned long gen;
    int busy;    /* workers still inside the current job */
};
static copy_pool g_pools[POOL_MAX_DEV];
static pthread_mutex_t g_pools_mu = PTHREAD_MUTEX_INITIALIZER;

static int device_numa_node(int dev) {
    char bdf[32];
    if (cudaDeviceGetPCIBusId(bdf, sizeof bdf, dev) != cudaSuccess) {
        cudaGetLastError();
        return -1;
    }
    for (char* p = bdf; *p; p++)
        if (*p >= 'A' && *p <= 'F') *p = (char)(*p - 'A' + 'a');
    char path[128];
    snprintf(path, sizeof path, "/sys/bus/pci/devices/%s/numa_node", bdf);
    FILE* f = fopen(path, "r");
    if (!f) return -1;
    int node = -1;
    if (fscanf(f, "%d", &node) != 1) node = -1;
    fclose(f);
    return node;
}

static int node_cpu_set(int node, cpu_set_t* set) {
    char path[128];
    snprintf(path, sizeof path, "/sys/devices/system/node/node%d/cpulist", node);
    FILE* f = fopen(path, "r");
    if (!f) return 0;
    CPU_ZERO(set);
    int a, b, any = 0;
    for (;;) {
        if (fscanf(f, "%d", &a) != 1) break;
        b = a;
        int ch = fgetc(f);
        if (ch == '-') {
            if (fscanf(f, "%d", &b) != 1) break;
            ch = fgetc(f);
        }
        for (int c = a; c <= b && c < CPU_SETSIZE; c++) {
            CPU_SET(c, set);
            any = 1;
        }
        if (ch != ',') break;
    }
    fclose(f);
    /* stay inside what the process may use */
    cpu_set_t allowed;
    if (any && sched_getaffinity(0, sizeof allowed, &allowed) == 0) {
        CPU_AND(set, set, &allowed);
        any = CPU_COUNT(set) > 0;
    }
    return any;
}

static void pool_run_slices(copy_pool* p) {
    for (;;) {
        const size_t off = __atomic_fetch_add(&p->next, POOL_SLICE, __ATOMIC_RELAXED);
        if (off >= p->bytes) break;
        const size_t n = p->bytes - off < POOL_SLICE ? p->bytes - off : POOL_SLICE;
        zxh_stream_copy(p->d + off, p->s + off, n);
    }
}

static void* pool_worker(void* arg) {
    copy_pool* p = (copy_pool*)arg;
    if (p->have_cpus) pthread_setaffinity_np(pthread_self(), sizeof p->cpus, &p->cpus);
    unsigned long seen = 0;
    pthread_mutex_lock(&p->mu);
    for (;;) {
        while (p->gen == seen) pthread_cond_wait(&p->cv_go, &p->mu);
        seen = p->gen;
        pthread_mutex_unlock(&p->mu);
        pool_run_slices(p);
        pthread_mutex_lock(&p->mu);
        if (--p->busy == 0) pthread_cond_signal(&p->cv_done);
    }
    return NULL;
}

static copy_pool* pool_for_device(int dev) {
    if (dev < 0 || dev >= POOL_MAX_DEV) dev = 0;
    copy_pool* p = &g_pools[dev];
    if (__atomic_load_n(&p->started, __ATOMIC_ACQUIRE)) return p;
    pthread_mutex_lock(&g_pools_mu);
    if (!p->started) {
        pthread_mutex_init(&p->job_mu, NULL);
        pthread_mutex_init(&p->mu, NULL);
        pthread_cond_init(&p->cv_go, NULL);
        pthread_cond_init(&p->cv_done, NULL);
        const int async_pool = dev >= POOL_MAX_DEV / 2;
        p->numa_node = device_numa_node(async_pool ? dev - POOL_MAX_DEV / 2 : dev);
        p->have_cpus = p->numa_node >= 0 && node_cpu_set(p->numa_node, &p->cpus);
        long ncpu = p->have_cpus ? CPU_COUNT(&p->cpus) : sysconf(_SC_NPROCESSORS_ONLN);
        const char* e = getenv("ZXC_B200_COPY_THREADS");
        /* per pool an eighth of the node's CPUs: more copy threads do not help -- the staged path is bound by host
         * memory traffic (9 bytes moved per 2 decoded), and PCIe DMA slows down when many threads compete with it */
        int want = e ? atoi(e) : (int)(ncpu / 8);
        if (want < 2) want = 2;
        if (want > POOL_MAX_THREADS) want = POOL_MAX_THREADS;
        p->n_threads = 0;
        for (int t = 0; t < want - (async_pool ? 0 : 1); t++) /* a synchronous job counts its caller as a member */
            if (pthread_create(&p->th[p->n_threads], NULL, pool_worker, p) == 0) p->n_threads++;
        __atomic_store_n(&p->started, 1, __ATOMIC_RELEASE);
    }
    pthread_mutex_unlock(&g_pools_mu);
    return p;
}

/* asynchronous variant on the device's second pool (workers only): pool_copy_begin returns at once,
 * pool_copy_end waits for the copy -- lets the caller's drain overlap its next fill */
static copy_pool* pool_copy_begin(int dev, void* dst, const void* src, size_t n) {
    if (dev < 0 || dev >= POOL_MAX_DEV / 2) dev = 0;
    copy_pool* p = pool_for_device(dev + POOL_MAX_DEV / 2);
    if (p->n_threads == 0 || n < ((size_t)2 << 20)) {
        zxh_stream_copy(dst, src, n);
        return NULL;
    }
    pthread_mutex_lock(&p->job_mu);
    pthread_mutex_lock(&p->mu);
    p->d = (u8*)dst;
    p->s = (const u8*)src;
    p->bytes = n;
    p->next = 0;
    p->busy = p->n_threads;
    p->gen++;
    pthread_cond_broadcast(&p->cv_go);
    pthread_mutex_unlock(&p->mu);
    return p;
}
static void pool_copy_end(copy_pool* p) {
    if (!p) return;
    pthread_mutex_lock(&p->mu);
    while (p->busy) pthread_cond_wait(&p->cv_done, &p->mu);
    pthread_mutex_unlock(&p->mu);
    pthread_mutex_unlock(&p->job_mu);
}

static void pool_memcpy(int dev, void* dst, const void* src, size_t n) {
    if (n < ((size_t)2 << 20)) {
        zxh_stream_copy(dst, src, n);
        return;
    }
    if (dev < 0 || dev >= POOL_MAX_DEV / 2) dev = 0;
    copy_pool* p = pool_for_device(dev);
    pthread_mutex_lock(&p->job_mu);
    pthread_mutex_lock(&p->mu);
    p->d = (u8*)dst;
    p->s = (const u8*)src;
    p->bytes = n;
    p->next = 0;
    p->busy = p->n_threads;
    p->gen++;
    pthread_cond_broadcast(&p->cv_go);
    pthread_mutex_unlock(&p->mu);
    pool_run_slices(p);
    pthread_mutex_lock(&p->mu);
    while (p->busy) pthread_cond_wait(&p->cv_done, &p->mu);
    pthread_mutex_unlock(&p->mu);
    pthread_mutex_unlock(&p->job_mu);
}

/* page-locked memory on the device's NUMA node: anonymous mapping, preferred-node policy, touched,
 * then registered with CUDA.  Falls back to cudaMallocHost when the node is unknown. */
struct pinned_buf {
    void* p;
    size_t bytes;
    int mapped; /* 1: mmap + cudaHostRegister, 0: cudaMallocHost */
};
static int pinned_alloc(pinned_buf* b, size_t bytes, int node) {
    b->p = NULL;
    b->bytes = bytes;
    b->mapped = 0;
    /* the driver allocates in the calling task's context: a preferred-node policy around the call puts the pages
     * next to the GPU; cudaMallocHost memory also DMAs faster than a registered 4 KiB-page mapping (measured) */
    int policy_set = 0;
#ifdef SYS_set_mempolicy
    if (node >= 0 && node < 64) {
        unsigned long mask = 1ul << node;
        policy_set = syscall(SYS_set_mempolicy, 1 /* MPOL_PREFERRED */, &mask, sizeof(mask) * 8) == 0;
    }
#endif
    const cudaError_t e = cudaMallocHost(&b->p, bytes);
#ifdef SYS_set_mempolicy
    if (policy_set) syscall(SYS_set_mempolicy, 0 /* MPOL_DEFAULT */, NULL, 0);
#endif
    if (e != cudaSuccess) {
        b->p = NULL;
        return ZXC_ERROR_MEMORY;
    }
    return ZXC_OK;
}
static void pinned_free(pinned_buf* b) {
    if (!b->p) return;
    if (b->mapped) {
        cudaHostUnregister(b->p);
        munmap(b->p, b->bytes);
    } else {
        cudaFreeHost(b->p);
    }
    b->p = NULL;
}

#define STAGE_SLOTS 4
#define EV_RING 8

struct zxg_ctx {
    cudaStream_t stream;
    void* buf[ZXG_BUF_COUNT];
    size_t cap[ZXG_BUF_COUNT];
    pinned_buf pinb[2];
    void* pin[2];
    cudaEvent_t pin_ev[2];
    unsigned long long* counter; /* [0..1] work counters, [2] deferred-job counter */
    unsigned long long* reduce_out; /* device: [0] first bad index, [1] byte sum (zxc_b200_reduce_status) */
    cudaStream_t s_h2d, s_d2h;   /* copy engines for the pipelined frame paths (lazily created) */
    cudaStream_t s_dec[STAGE_SLOTS]; /* staged path: chunk decodes overlap (a 512-block launch is latency-bound) */
    cudaEvent_t ev_ring[EV_RING]; /* reused by the pipelines: no event is created per chunk */
    pinned_buf st_in[STAGE_SLOTS], st_out[STAGE_SLOTS]; /* staging for pageable callers (lazily allocated) */
    cudaEvent_t st_ev_in[STAGE_SLOTS], st_ev_dec[STAGE_SLOTS], st_ev_out[STAGE_SLOTS];
    int st_ready;
    struct zxg_ctx* next;
    int device;
    int numa_node;
    int sm_count;
    int trimmed; /* idle and already cut back by zxg_release */
};
static zxg_ctx* g_free_list = NULL;

static void init_once(void) {
    int n = 0;
    const cudaError_t e = cudaGetDeviceCount(&n);
    if (e != cudaSuccess || n <= 0) {
        fprintf(stderr,
                "libzxc (CUDA build): no usable CUDA device (%s); this library has no CPU codec, "
                "codec entry points return ZXC_B200_ERROR_NO_DEVICE\n",
                e != cudaSuccess ? cudaGetErrorString(e) : "device count 0");
        g_init_rc = ZXC_B200_ERROR_NO_DEVICE;
        return;
    }
    int dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceProp prop;
    if (cudaGetDeviceProperties(&prop, dev) != cudaSuccess) {
        g_init_rc = ZXC_B200_ERROR_CUDA;
        return;
    }
    g_sm_count = prop.multiProcessorCount;
    g_init_rc = ZXC_OK;
}

extern "C" int zxg_init(void) {
    pthread_once(&g_once, init_once);
    return g_init_rc;
}

extern "C" int zxc_b200_device_count(void) {
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess) return 0;
    return n;
}

extern "C" uint64_t zxc_b200_launch_count(void) { return g_launches; }

extern "C" int zxc_b200_decode_occupancy(int* lean, int* general) {
    if (zxg_init() != ZXC_OK) return ZXC_B200_ERROR_CUDA;
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(lean, zxc_decode_kernel<false, false, false, true>, CTA_THREADS,
                                                      LEAN_SMEM_BYTES) != cudaSuccess ||
        cudaOccupancyMaxActiveBlocksPerMultiprocessor(general, zxc_decode_kernel<false, true, false, false>, CTA_THREADS,
                                                      DECODE_SMEM_BYTES) != cudaSuccess)
        return ZXC_B200_ERROR_CUDA;
    return ZXC_OK;
}

#if ZXC_TRACE
/* traced build only: copies the current device's phase-trace rows (TRACE_ROWS x TRACE_SLOTS counters) to `host` and
 * zeroes them; returns the number of counters */
extern "C" ZXC_EXPORT int zxc_b200_trace_read(unsigned long long* host) {
    const size_t bytes = sizeof(unsigned long long) * TRACE_ROWS * TRACE_SLOTS;
    if (cudaDeviceSynchronize() != cudaSuccess) return -1;
    if (cudaMemcpyFromSymbol(host, zxc_trace_acc, bytes) != cudaSuccess) return -1;
    void* d = 0;
    if (cudaGetSymbolAddress(&d, zxc_trace_acc) != cudaSuccess || cudaMemset(d, 0, bytes) != cudaSuccess) return -1;
    if (cudaDeviceSynchronize() != cudaSuccess) return -1;
    return TRACE_ROWS * TRACE_SLOTS;
}
#endif

extern "C" int zxg_current_device(void) {
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess) {
        cudaGetLastError();
        return 0;
    }
    return dev;
}
extern "C" int zxg_device_count(void) { return zxc_b200_device_count(); }
extern "C" int zxg_set_device(int dev) {
    if (cudaSetDevice(dev) != cudaSuccess) {
        cudaGetLastError();
        return ZXC_B200_ERROR_CUDA;
    }
    return ZXC_OK;
}

extern "C" zxg_ctx* zxg_create(void) {
    if (zxg_init() != ZXC_OK) return NULL;
    zxg_ctx* c = (zxg_ctx*)calloc(1, sizeof(zxg_ctx));
    if (!c) return NULL;
    cudaGetDevice(&c->device);
    if (cudaStreamCreateWithFlags(&c->stream, cudaStreamNonBlocking) != cudaSuccess ||
        cudaMalloc((void**)&c->counter, 32 * sizeof(unsigned long long)) != cudaSuccess) {
        free(c);
        return NULL;
    }
    c->reduce_out = c->counter + 28;
    c->numa_node = device_numa_node(c->device);
    int smc = 0;
    if (cudaDeviceGetAttribute(&smc, cudaDevAttrMultiProcessorCount, c->device) != cudaSuccess || smc <= 0) smc = g_sm_count;
    c->sm_count = smc;
    return c;
}

extern "C" void zxg_destroy(zxg_ctx* c) {
    if (!c) return;
    cudaStreamSynchronize(c->stream);
    for (int i = 0; i < ZXG_BUF_COUNT; i++)
        if (c->buf[i]) cudaFree(c->buf[i]);
    for (int i = 0; i < 2; i++) {
        pinned_free(&c->pinb[i]);
        if (c->pin_ev[i]) cudaEventDestroy(c->pin_ev[i]);
    }
    for (int i = 0; i < STAGE_SLOTS; i++) {
        pinned_free(&c->st_in[i]);
        pinned_free(&c->st_out[i]);
        if (c->st_ev_in[i]) cudaEventDestroy(c->st_ev_in[i]);
        if (c->st_ev_dec[i]) cudaEventDestroy(c->st_ev_dec[i]);
        if (c->st_ev_out[i]) cudaEventDestroy(c->st_ev_out[i]);
    }
    for (int i = 0; i < EV_RING; i++)
        if (c->ev_ring[i]) cudaEventDestroy(c->ev_ring[i]);
    cudaFree(c->counter);
    for (int i = 0; i < STAGE_SLOTS; i++)
        if (c->s_dec[i]) cudaStreamDestroy(c->s_dec[i]);
    if (c->s_h2d) cudaStreamDestroy(c->s_h2d);
    if (c->s_d2h) cudaStreamDestroy(c->s_d2h);
    cudaStreamDestroy(c->stream);
    free(c);
}

extern "C" zxg_ctx* zxg_acquire(void) {
    if (zxg_init() != ZXC_OK) return NULL;
    int dev = 0;
    cudaGetDevice(&dev);
    pthread_mutex_lock(&g_pool_mu);
    zxg_ctx** pp = &g_free_list;
    while (*pp && (*pp)->device != dev) pp = &(*pp)->next;
    zxg_ctx* c = *pp;
    if (c) *pp = c->next;
    pthread_mutex_unlock(&g_pool_mu);
    if (c) {
        c->next = NULL;
        return c;
    }
    return zxg_create();
}

/* Gives back what an idle context holds beyond `keep` bytes per buffer (and its staging slots). */
static void ctx_trim(zxg_ctx* c, size_t keep) {
    cudaStreamSynchronize(c->stream);
    for (int i = 0; i < ZXG_BUF_COUNT; i++)
        if (c->buf[i] && c->cap[i] > keep) {
            cudaFree(c->buf[i]);
            c->buf[i] = NULL;
            c->cap[i] = 0;
        }
    for (int i = 0; i < STAGE_SLOTS; i++) {
        pinned_free(&c->st_in[i]);
        pinned_free(&c->st_out[i]);
    }
}

/* The free list keeps contexts warm: the two most recently released contexts of a device keep their buffers (a
 * caller that decodes frame after frame should not pay cudaMalloc each time); older idle ones -- left behind by a
 * burst of concurrent callers -- are trimmed to POOL_KEEP_BYTES per buffer so that one multi-GiB frame does not pin
 * several GiB of HBM per past thread for the life of the process. */
#define POOL_WARM_PER_DEVICE 2
#define POOL_KEEP_BYTES ((size_t)64 << 20)
extern "C" void zxg_release(zxg_ctx* c) {
    if (!c) return;
    pthread_mutex_lock(&g_pool_mu);
    c->next = g_free_list;
    g_free_list = c;
    int seen = 0;
    for (zxg_ctx* q = g_free_list; q; q = q->next) {
        if (q->device != c->device) continue;
        if (++seen > POOL_WARM_PER_DEVICE && !q->trimmed) {
            ctx_trim(q, POOL_KEEP_BYTES);
            q->trimmed = 1;
        }
    }
    c->trimmed = 0;
    pthread_mutex_unlock(&g_pool_mu);
}

extern "C" void* zxg_buffer(zxg_ctx* c, int which, size_t bytes) {
    if (bytes == 0) bytes = 16;
    if (c->cap[which] >= bytes) return c->buf[which];
    if (c->buf[which]) {
        cudaStreamSynchronize(c->stream);
        cudaFree(c->buf[which]);
        c->buf[which] = NULL;
        c->cap[which] = 0;
    }
    size_t want = bytes + (bytes >> 3) + 256; /* slack against regrowth */
    void* p = NULL;
    if (cudaMalloc(&p, want) != cudaSuccess) {
        want = bytes;
        if (cudaMalloc(&p, want) != cudaSuccess) return NULL;
    }
    c->buf[which] = p;
    c->cap[which] = want;
    return p;
}

extern "C" void* zxg_stream(zxg_ctx* c) { return (void*)c->stream; }

extern "C" int zxg_sync(zxg_ctx* c) {
    return cudaStreamSynchronize(c->stream) == cudaSuccess ? ZXC_OK : ZXC_B200_ERROR_CUDA;
}

static int host_is_pinned(const void* p) {
    cudaPointerAttributes a;
    if (cudaPointerGetAttributes(&a, p) != cudaSuccess) {
        cudaGetLastError();
        return 0;
    }
    return a.type == cudaMemoryTypeHost || a.type == cudaMemoryTypeManaged;
}

static int ensure_pins(zxg_ctx* c) {
    for (int i = 0; i < 2; i++) {
        if (!c->pin[i]) {
            if (pinned_alloc(&c->pinb[i], PIN_CHUNK, c->numa_node) != ZXC_OK) return ZXC_ERROR_MEMORY;
            c->pin[i] = c->pinb[i].p;
            if (cudaEventCreateWithFlags(&c->pin_ev[i], cudaEventDisableTiming) != cudaSuccess)
                return ZXC_B200_ERROR_CUDA;
        }
    }
    return ZXC_OK;
}

extern "C" int zxg_h2d(zxg_ctx* c, void* d_dst, const void* h_src, size_t bytes) {
    if (bytes == 0) return ZXC_OK;
    if (host_is_pinned(h_src) || bytes <= (64u << 10)) {
        return cudaMemcpyAsync(d_dst, h_src, bytes, cudaMemcpyHostToDevice, c->stream) == cudaSuccess
                   ? ZXC_OK : ZXC_B200_ERROR_CUDA;
    }
    const int rc = ensure_pins(c);
    if (rc != ZXC_OK) return rc;
    size_t done = 0;
    int slot = 0;
    while (done < bytes) {
        const size_t n = bytes - done < PIN_CHUNK ? bytes - done : PIN_CHUNK;
        cudaEventSynchronize(c->pin_ev[slot]); /* previous use of this bounce buffer */
        pool_memcpy(c->device, c->pin[slot], (const u8*)h_src + done, n);
        if (cudaMemcpyAsync((u8*)d_dst + done, c->pin[slot], n, cudaMemcpyHostToDevice, c->stream) != cudaSuccess)
            return ZXC_B200_ERROR_CUDA;
        cudaEventRecord(c->pin_ev[slot], c->stream);
        done += n;
        slot ^= 1;
    }
    return ZXC_OK;
}

extern "C" int zxg_d2h(zxg_ctx* c, void* h_dst, const void* d_src, size_t bytes) {
    if (bytes == 0) return ZXC_OK;
    if (host_is_pinned(h_dst)) {
        if (cudaMemcpyAsync(h_dst, d_src, bytes, cudaMemcpyDeviceToHost, c->stream) != cudaSuccess)
            return ZXC_B200_ERROR_CUDA;
        return zxg_sync(c);
    }
    const int rc = ensure_pins(c);
    if (rc != ZXC_OK) return rc;
    /* double buffer: while chunk k is copied out of its bounce buffer, chunk k+1 is in flight */
    const size_t nchunks = (bytes + PIN_CHUNK - 1) / PIN_CHUNK;
    for (size_t k = 0; k <= nchunks; k++) {
        if (k < nchunks) { /* issue chunk k into slot k&1 (its previous contents were drained at k-1) */
            const size_t off = k * PIN_CHUNK;
            const size_t n = bytes - off < PIN_CHUNK ? bytes - off : PIN_CHUNK;
            if (cudaMemcpyAsync(c->pin[k & 1], (const u8*)d_src + off, n, cudaMemcpyDeviceToHost, c->stream) != cudaSuccess)
                return ZXC_B200_ERROR_CUDA;
            cudaEventRecord(c->pin_ev[k & 1], c->stream);
        }
        if (k > 0) { /* drain chunk k-1 */
            const size_t off = (k - 1) * PIN_CHUNK;
            const size_t n = bytes - off < PIN_CHUNK ? bytes - off : PIN_CHUNK;
            if (cudaEventSynchronize(c->pin_ev[(k - 1) & 1]) != cudaSuccess) return ZXC_B200_ERROR_CUDA;
            pool_memcpy(c->device, (u8*)h_dst + off, c->pin[(k - 1) & 1], n);
        }
    }
    return ZXC_OK;
}

/* the larger of the lean and the general instance's CTAs per SM: the decode grid and the per-warp scratch are sized
 * for it (the lean launch comes first and decodes nearly every block) */
#define DECODE_CTAS_MAX (LEAN_CTAS_PER_SM > CTAS_PER_SM ? LEAN_CTAS_PER_SM : CTAS_PER_SM)

/* resident decode CTAs per SM: DECODE_CTAS_MAX unless ZXC_B200_DECODE_CTAS (1..DECODE_CTAS_MAX) says fewer --
 * a tuning knob: fewer warps keep fewer 64 KiB output windows alive in L2 (DESIGN.md section 9) */
static u32 decode_ctas_per_sm(void) {
    static int cached = 0;
    if (cached == 0) {
        const char* e = getenv("ZXC_B200_DECODE_CTAS");
        const int v = e ? atoi(e) : 0;
        cached = (v >= 1 && v <= (int)DECODE_CTAS_MAX) ? v : (int)DECODE_CTAS_MAX;
    }
    return (u32)cached;
}

static int grid_for(u32 n_jobs) {
    const u32 ctas_needed = (n_jobs + WARPS_PER_CTA - 1) / WARPS_PER_CTA;
    const u32 resident = (u32)(g_sm_count > 0 ? g_sm_count : 132) * decode_ctas_per_sm();
    return (int)(ctas_needed < resident ? ctas_needed : resident);
}

/* per-warp scratch for expanded literal sections; 256 bytes of lead-in so word loads may start below it */
static u32 scratch_stride_for(u32 block_size) { return scr_stride(block_size); }

#define SCRATCH_TAIL (sizeof(unsigned long long) * 4)
#define DEFER_CAP (1u << 16) /* listed deferred jobs; beyond that the second launch scans the status array */

extern "C" size_t zxc_b200_decode_scratch_size(uint32_t block_size) {
    if (zxg_init() != ZXC_OK) return 0;
    const size_t warps = (size_t)g_sm_count * DECODE_CTAS_MAX * WARPS_PER_CTA;
    const size_t n = warps * scratch_stride_for(block_size) + 512; /* room to align the regions behind it to 256 bytes */
    return n + (size_t)DEFER_CAP * 4 + SCRATCH_TAIL;
}

/* d_counter: three 64-bit work counters, zeroed here unless `preset` (then the caller has set them already: the
 * device-planned decode starts the claims at its first real job, zxc_dplan.cuh) */
static int launch_decode(const void* d_src, void* d_dst, const zxc_b200_job_t* d_jobs, u32 n_jobs,
                         i32* d_status, const void* d_dict, u32 dict_size, const void* d_dict_huf,
                         void* d_scratch, size_t scratch_size, u32 block_size, int verify,
                         unsigned long long* d_counter, cudaStream_t st, int preset) {
    if (n_jobs == 0) return ZXC_OK;
    DecodeParams P;
    P.src = (const u8*)d_src;
    P.dst = (u8*)d_dst;
    P.jobs = d_jobs;
    P.status = d_status;
    P.dict = (const u8*)d_dict;
    P.dict_huf = (const u8*)d_dict_huf;
    P.scratch = (u8*)d_scratch;
    P.counter = d_counter;
    P.n_jobs = n_jobs;
    P.dict_size = d_dict ? dict_size : 0;
    P.scratch_stride = scratch_stride_for(block_size);
    P.flags = verify ? FLAG_VERIFY : 0;
    {
        static int units_mode = -2; /* ZXC_B200_UNITS: 1 = always, 0 = never, unset = by measured rule */
        if (units_mode == -2) {
            const char* e = getenv("ZXC_B200_UNITS");
            units_mode = e ? (e[0] == '1' ? 1 : 0) : -1;
        }
        if (units_mode == 1) P.flags |= FLAG_UNITS_ON;
        if (units_mode == 0) P.flags |= FLAG_UNITS_OFF;
    }
    /* The output-centric body (zxc_decode_units.cuh) was the faster one for dictionary decodes of small blocks while the
     * sequence-centric body copied dictionary sources byte by byte.  Since that body reads them as ordinary global
     * sources and copies long items as balanced chunks it wins there too (DESIGN.md), so the unit walk runs only on
     * request (ZXC_B200_UNITS=1). */
    const bool units = (P.flags & FLAG_UNITS_ON) != 0;
    P.block_cap = block_size;
    int grid = grid_for(n_jobs);
    const size_t warp_scratch = (size_t)grid * WARPS_PER_CTA * P.scratch_stride;
    if (warp_scratch > scratch_size) return ZXC_ERROR_MEMORY;
    if (!preset && cudaMemsetAsync(d_counter, 0, 3 * sizeof(unsigned long long), st) != cudaSuccess)
        return ZXC_B200_ERROR_CUDA;
    /* deferred-job list behind the per-warp scratch; its counter is the third work counter.  A scratch too small for it
     * leaves the list empty: the second launch scans the status array. */
    const size_t off =(warp_scratch + 255) & ~(size_t)255;
    P.defer_count = (u32*)(d_counter + 2);
    P.defer_cap = off + (size_t)DEFER_CAP * 4 <= scratch_size ? DEFER_CAP : 0u;
    P.defer_list = (u32*)((u8*)d_scratch + off);
    /* the dictionary-free instance carries neither the dictionary pointer nor its source classification (zxc_decode.cuh) */
    const bool has_dict = P.dict != NULL && P.dict_size != 0;
    if (!verify && !units) {
        /* launch 1: the lean instance decodes the RAW blocks and the GLO blocks without Huffman sections and lists the
         * rest; launch 2 below: the general instance decodes the listed jobs (its warps exit at once when there are none) */
#ifdef LEAN_CARVEOUT
        /* development: the shared-memory share of the unified L1 / shared array, in percent, as a hint to the driver */
        static int carveout_done = 0;
        if (!carveout_done) {
            cudaFuncSetAttribute(zxc_decode_kernel<false, false, true, true>,
                                 cudaFuncAttributePreferredSharedMemoryCarveout, LEAN_CARVEOUT);
            cudaFuncSetAttribute(zxc_decode_kernel<false, false, false, true>,
                                 cudaFuncAttributePreferredSharedMemoryCarveout, LEAN_CARVEOUT);
            carveout_done = 1;
        }
#endif
        const u32 lean_smem = has_dict ? DECODE_SMEM_BYTES + LEAN_SMEM_PAD : LEAN_SMEM_BYTES; /* + look-ahead slots */
        if (has_dict) zxc_decode_kernel<false, false, true, true><<<grid, CTA_THREADS, lean_smem, st>>>(P);
        else zxc_decode_kernel<false, false, false, true><<<grid, CTA_THREADS, lean_smem, st>>>(P);
        __atomic_add_fetch(&g_launches, 1, __ATOMIC_RELAXED);
        if (cudaGetLastError() != cudaSuccess) return ZXC_B200_ERROR_CUDA;
        P.flags |= FLAG_DEFERRED;
        P.counter = d_counter + 1;
    }
    /* the general instances run at CTAS_PER_SM: a grid of the lean instance's size would leave its extra CTAs waiting
     * for a slot and claiming what is left at the end */
    {
        const int resident = (g_sm_count > 0 ? g_sm_count : 132) * (int)CTAS_PER_SM;
        if (grid > resident) grid = resident;
    }
    if (P.flags & FLAG_DEFERRED) {
        if (has_dict) zxc_decode_kernel<false, true, true, false><<<grid, CTA_THREADS, DECODE_SMEM_BYTES, st>>>(P);
        else zxc_decode_kernel<false, true, false, false><<<grid, CTA_THREADS, DECODE_SMEM_BYTES, st>>>(P);
    } else if (units) {
        if (has_dict) zxc_decode_kernel<true, false, true, false><<<grid, CTA_THREADS, DECODE_SMEM_BYTES, st>>>(P);
        else zxc_decode_kernel<true, false, false, false><<<grid, CTA_THREADS, DECODE_SMEM_BYTES, st>>>(P);
    } else {
        if (has_dict) zxc_decode_kernel<false, false, true, false><<<grid, CTA_THREADS, DECODE_SMEM_BYTES, st>>>(P);
        else zxc_decode_kernel<false, false, false, false><<<grid, CTA_THREADS, DECODE_SMEM_BYTES, st>>>(P);
    }
    __atomic_add_fetch(&g_launches, 1, __ATOMIC_RELAXED);
    return cudaGetLastError() == cudaSuccess ? ZXC_OK : ZXC_B200_ERROR_CUDA;
}

/* device scratch one launch over n_jobs blocks needs (without the counter tail) */
static size_t launch_scratch_bytes(u32 n_jobs, u32 block_size) {
    size_t n = (size_t)grid_for(n_jobs) * WARPS_PER_CTA * scratch_stride_for(block_size);
    n = (n + 255) & ~(size_t)255;
    return n + (size_t)DEFER_CAP * 4 + 256;
}

extern "C" int zxc_b200_decode_blocks(const void* d_src, void* d_dst, const zxc_b200_job_t* d_jobs,
                                      uint32_t n_jobs, int32_t* d_status, const void* d_dict,
                                      uint32_t dict_size, const void* d_dict_huf, void* d_scratch,
                                      size_t scratch_size, uint32_t block_size, int verify_checksums,
                                      void* stream) {
    const int rc = zxg_init();
    if (rc != ZXC_OK) return rc;
    if (!d_src || !d_dst || !d_jobs || !d_status || !d_scratch) return ZXC_ERROR_NULL_INPUT;
    if (scratch_size < SCRATCH_TAIL) return ZXC_ERROR_MEMORY;
    /* the work counters live in the last 32 bytes of the caller's scratch */
    const size_t usable = (scratch_size - SCRATCH_TAIL) & ~(size_t)7;
    unsigned long long* counter = (unsigned long long*)((u8*)d_scratch + usable);
    return launch_decode(d_src, d_dst, d_jobs, n_jobs, d_status, d_dict, dict_size, d_dict_huf,
                         d_scratch, usable, block_size, verify_checksums, counter, (cudaStream_t)stream, 0);
}

/* one 16-byte result slot per device, allocated on first use and kept: no cudaMalloc / cudaFree per call */
static unsigned long long* g_reduce_dev[POOL_MAX_DEV];
static pthread_mutex_t g_reduce_mu = PTHREAD_MUTEX_INITIALIZER;

extern "C" int64_t zxc_b200_reduce_status(const int32_t* d_status, const zxc_b200_job_t* d_jobs,
                                          uint32_t n_jobs, void* stream) {
    const int rc = zxg_init();
    if (rc != ZXC_OK) return rc;
    if (n_jobs == 0) return 0;
    cudaStream_t st = (cudaStream_t)stream;
    int dev = 0;
    cudaGetDevice(&dev);
    if (dev < 0 || dev >= POOL_MAX_DEV) dev = 0;
    pthread_mutex_lock(&g_reduce_mu);
    if (!g_reduce_dev[dev] && cudaMalloc((void**)&g_reduce_dev[dev], 16) != cudaSuccess) {
        g_reduce_dev[dev] = NULL;
        pthread_mutex_unlock(&g_reduce_mu);
        return ZXC_ERROR_MEMORY;
    }
    unsigned long long* d_out = g_reduce_dev[dev];
    const unsigned long long init[2] = {~0ull, 0ull};
    cudaMemcpyAsync(d_out, init, 16, cudaMemcpyHostToDevice, st);
    zxc_reduce_kernel<<<(n_jobs + 255) / 256, 256, 0, st>>>(d_status, d_jobs, n_jobs, d_out);
    __atomic_add_fetch(&g_launches, 1, __ATOMIC_RELAXED);
    unsigned long long h[2] = {0, 0};
    cudaMemcpyAsync(h, d_out, 16, cudaMemcpyDeviceToHost, st);
    const cudaError_t e = cudaStreamSynchronize(st);
    int64_t ret;
    if (e != cudaSuccess) {
        ret = ZXC_B200_ERROR_CUDA;
    } else if (h[0] != ~0ull) {
        i32 s = 0;
        cudaMemcpy(&s, d_status + h[0], 4, cudaMemcpyDeviceToHost);
        ret = s < 0 ? s : ZXC_ERROR_CORRUPT_DATA;
    } else {
        ret = (int64_t)h[1];
    }
    pthread_mutex_unlock(&g_reduce_mu);
    return ret;
}

/* A decode's dictionary into the context's ZXG_BUF_DICT, its 128-byte literal table (when given) right behind it;
 * both device pointers stay NULL without a dictionary. */
static int upload_dict(zxg_ctx* c, const void* h_dict, u32 dict_size, const void* h_dict_huf, u8** d_dict,
                       u8** d_huf) {
    *d_dict = NULL;
    *d_huf = NULL;
    if (!h_dict || !dict_size) return ZXC_OK;
    *d_dict = (u8*)zxg_buffer(c, ZXG_BUF_DICT, (size_t)dict_size + 128);
    if (!*d_dict) return ZXC_ERROR_MEMORY;
    int rc = zxg_h2d(c, *d_dict, h_dict, dict_size);
    if (rc == ZXC_OK && h_dict_huf) {
        *d_huf = *d_dict + dict_size;
        rc = zxg_h2d(c, *d_huf, h_dict_huf, 128);
    }
    return rc;
}

extern "C" int zxg_decode_jobs(zxg_ctx* c, const void* d_src, void* d_dst, const zxc_b200_job_t* h_jobs,
                               uint32_t n_jobs, int32_t* h_status, const void* h_dict, uint32_t dict_size,
                               const void* h_dict_huf, uint32_t block_size, int verify_checksums) {
    if (n_jobs == 0) return ZXC_OK;
    zxc_b200_job_t* d_jobs = (zxc_b200_job_t*)zxg_buffer(c, ZXG_BUF_JOBS, (size_t)n_jobs * sizeof(zxc_b200_job_t));
    i32* d_status = (i32*)zxg_buffer(c, ZXG_BUF_STATUS, (size_t)n_jobs * sizeof(i32));
    const size_t scratch_size = launch_scratch_bytes(n_jobs, block_size);
    void* d_scratch = zxg_buffer(c, ZXG_BUF_SCRATCH, scratch_size);
    if (!d_jobs || !d_status || !d_scratch) return ZXC_ERROR_MEMORY;
    u8 *d_dict, *d_huf;
    int rc = upload_dict(c, h_dict, dict_size, h_dict_huf, &d_dict, &d_huf);
    if (rc != ZXC_OK) return rc;
    rc = zxg_h2d(c, d_jobs, h_jobs, (size_t)n_jobs * sizeof(zxc_b200_job_t));
    if (rc != ZXC_OK) return rc;
    rc = launch_decode(d_src, d_dst, d_jobs, n_jobs, d_status, d_dict, dict_size, d_huf, d_scratch,
                       scratch_size, block_size, verify_checksums, c->counter, c->stream, 0);
    if (rc != ZXC_OK) return rc;
    if (cudaMemcpyAsync(h_status, d_status, (size_t)n_jobs * sizeof(i32), cudaMemcpyDeviceToHost, c->stream) != cudaSuccess)
        return ZXC_B200_ERROR_CUDA;
    if (cudaStreamSynchronize(c->stream) != cudaSuccess) {
        fprintf(stderr, "libzxc (CUDA build): decode kernel failed: %s\n", cudaGetErrorString(cudaGetLastError()));
        return ZXC_B200_ERROR_CUDA;
    }
    return ZXC_OK;
}


/* ------------------------------------------------------------------------- */
/* Pipelined frame decode for page-locked host buffers: the frame is cut into  */
/* chunks of whole blocks; chunk k's H2D copy, chunk k-1's decode and chunk     */
/* k-2's D2H copy run concurrently on three streams (both PCIe directions and   */
/* the SMs busy at once).  Pageable buffers take the staged path instead.       */
/* ------------------------------------------------------------------------- */
extern "C" int zxg_host_pinned(const void* p) { return host_is_pinned(p); }

extern "C" int zxg_decode_pipelined(zxg_ctx* c, const uint8_t* h_src, uint64_t src_lo, uint64_t src_hi,
                                    uint8_t* h_dst, uint64_t produced, const zxc_b200_job_t* h_jobs,
                                    uint32_t n_jobs, int32_t* h_status, const void* h_dict, uint32_t dict_size,
                                    const void* h_dict_huf, uint32_t block_size, int verify_checksums) {
    if (n_jobs == 0) return ZXC_OK;
    if (!c->s_h2d && cudaStreamCreateWithFlags(&c->s_h2d, cudaStreamNonBlocking) != cudaSuccess) return ZXC_B200_ERROR_CUDA;
    if (!c->s_d2h && cudaStreamCreateWithFlags(&c->s_d2h, cudaStreamNonBlocking) != cudaSuccess) return ZXC_B200_ERROR_CUDA;
    u8* d_in = (u8*)zxg_buffer(c, ZXG_BUF_IN, (size_t)(src_hi - src_lo) + 16);
    u8* d_out = (u8*)zxg_buffer(c, ZXG_BUF_OUT, (size_t)produced + 16);
    zxc_b200_job_t* d_jobs = (zxc_b200_job_t*)zxg_buffer(c, ZXG_BUF_JOBS, (size_t)n_jobs * sizeof(zxc_b200_job_t));
    i32* d_status = (i32*)zxg_buffer(c, ZXG_BUF_STATUS, (size_t)n_jobs * sizeof(i32));
    const size_t scratch_size = launch_scratch_bytes(n_jobs, block_size);
    void* d_scratch = zxg_buffer(c, ZXG_BUF_SCRATCH, scratch_size);
    if (!d_in || !d_out || !d_jobs || !d_status || !d_scratch) return ZXC_ERROR_MEMORY;
    u8 *d_dict, *d_huf;
    int rc = upload_dict(c, h_dict, dict_size, h_dict_huf, &d_dict, &d_huf);
    if (rc != ZXC_OK) return rc;
    /* the job table goes up chunk by chunk, just ahead of each launch: one copy of the whole table (24 MB for a million
     * 4 KiB records, staged synchronously by the driver when the table is pageable) would sit in front of the first
     * H2D of payload */
    const uint64_t chunk_target = (uint64_t)64 << 20; /* decoded bytes per pipeline stage */
    for (int i = 0; i < EV_RING; i++)
        if (!c->ev_ring[i] && cudaEventCreateWithFlags(&c->ev_ring[i], cudaEventDisableTiming) != cudaSuccess)
            return ZXC_B200_ERROR_CUDA;
    uint32_t j0 = 0, chunk_no = 0;
    while (j0 < n_jobs && rc == ZXC_OK) {
        /* events are recycled: a wait refers to the record that preceded it, so reuse is safe */
        const cudaEvent_t ev_in = c->ev_ring[(2u * chunk_no) % EV_RING], ev_dec = c->ev_ring[(2u * chunk_no + 1u) % EV_RING];
        chunk_no++;
        uint32_t j1 = j0;
        uint64_t acc = 0;
        while (j1 < n_jobs && acc < chunk_target) acc += h_jobs[j1++].dst_cap;
        const uint64_t s0 = h_jobs[j0].src_off, s1 = h_jobs[j1 - 1].src_off + h_jobs[j1 - 1].src_len;
        const uint64_t o0 = h_jobs[j0].dst_off, o1 = h_jobs[j1 - 1].dst_off + h_jobs[j1 - 1].dst_cap;
        if (cudaMemcpyAsync(d_in + (s0 - src_lo), h_src + s0, (size_t)(s1 - s0), cudaMemcpyHostToDevice, c->s_h2d) != cudaSuccess)
            rc = ZXC_B200_ERROR_CUDA;
        cudaEventRecord(ev_in, c->s_h2d);
        if (cudaMemcpyAsync(d_jobs + j0, h_jobs + j0, (size_t)(j1 - j0) * sizeof(zxc_b200_job_t), cudaMemcpyHostToDevice,
                            c->stream) != cudaSuccess)
            rc = ZXC_B200_ERROR_CUDA;
        cudaStreamWaitEvent(c->stream, ev_in, 0);
        if (rc == ZXC_OK)
            rc = launch_decode(d_in - src_lo, d_out, d_jobs + j0, j1 - j0, d_status + j0, d_dict, dict_size, d_huf,
                               d_scratch, scratch_size, block_size, verify_checksums, c->counter, c->stream, 0);
        cudaEventRecord(ev_dec, c->stream);
        cudaStreamWaitEvent(c->s_d2h, ev_dec, 0);
        if (rc == ZXC_OK &&
            cudaMemcpyAsync(h_dst + o0, d_out + o0, (size_t)(o1 - o0), cudaMemcpyDeviceToHost, c->s_d2h) != cudaSuccess)
            rc = ZXC_B200_ERROR_CUDA;
        j0 = j1;
    }
    if (rc == ZXC_OK &&
        cudaMemcpyAsync(h_status, d_status, (size_t)n_jobs * sizeof(i32), cudaMemcpyDeviceToHost, c->stream) != cudaSuccess)
        rc = ZXC_B200_ERROR_CUDA;
    const cudaError_t e1 = cudaStreamSynchronize(c->stream);
    const cudaError_t e2 = cudaStreamSynchronize(c->s_d2h);
    const cudaError_t e3 = cudaStreamSynchronize(c->s_h2d);
    if (e1 != cudaSuccess || e2 != cudaSuccess || e3 != cudaSuccess) {
        fprintf(stderr, "libzxc (CUDA build): pipelined decode failed: %s\n", cudaGetErrorString(cudaGetLastError()));
        return ZXC_B200_ERROR_CUDA;
    }
    return rc;
}


/* ------------------------------------------------------------------------- */
/* Staged frame decode for ordinary (pageable) caller memory: the same three     */
/* streams as zxg_decode_pipelined, with pinned bounce buffers either side.  The  */
/* host thread fills input slot k (copy pool, or the caller's read_at), queues    */
/* H2D / decode / D2H for chunk k, then drains output slot k-2 into the caller's   */
/* buffer while the GPU works -- so PCIe in, the SMs, PCIe out and the host copies */
/* all overlap.  Decoded coordinates: job dst offsets; [clip_lo, clip_hi) of them  */
/* is what the caller wants at h_dst (ranges start and end inside blocks).         */
/* ------------------------------------------------------------------------- */
#define STAGE_OUT ((size_t)32 << 20)
#define STAGE_IN (STAGE_OUT + ((size_t)1 << 20))

static int staged_ready(zxg_ctx* c) {
    if (c->st_ready) return ZXC_OK;
    for (int i = 0; i < STAGE_SLOTS; i++) {
        if (!c->st_in[i].p && pinned_alloc(&c->st_in[i], STAGE_IN, c->numa_node) != ZXC_OK) return ZXC_ERROR_MEMORY;
        if (!c->st_out[i].p && pinned_alloc(&c->st_out[i], STAGE_OUT, c->numa_node) != ZXC_OK) return ZXC_ERROR_MEMORY;
        if (!c->st_ev_in[i] && cudaEventCreateWithFlags(&c->st_ev_in[i], cudaEventDisableTiming) != cudaSuccess) return ZXC_B200_ERROR_CUDA;
        if (!c->st_ev_dec[i] && cudaEventCreateWithFlags(&c->st_ev_dec[i], cudaEventDisableTiming) != cudaSuccess) return ZXC_B200_ERROR_CUDA;
        if (!c->st_ev_out[i] && cudaEventCreateWithFlags(&c->st_ev_out[i], cudaEventDisableTiming) != cudaSuccess) return ZXC_B200_ERROR_CUDA;
    }
    if (!c->s_h2d && cudaStreamCreateWithFlags(&c->s_h2d, cudaStreamNonBlocking) != cudaSuccess) return ZXC_B200_ERROR_CUDA;
    if (!c->s_d2h && cudaStreamCreateWithFlags(&c->s_d2h, cudaStreamNonBlocking) != cudaSuccess) return ZXC_B200_ERROR_CUDA;
    for (int i = 0; i < STAGE_SLOTS; i++)
        if (!c->s_dec[i] && cudaStreamCreateWithFlags(&c->s_dec[i], cudaStreamNonBlocking) != cudaSuccess) return ZXC_B200_ERROR_CUDA;
    c->st_ready = 1;
    return ZXC_OK;
}

struct staged_chunk {
    uint32_t j0, j1;
    uint64_t s0, s1;   /* source byte range */
    uint64_t c0, c1;   /* clipped decoded range delivered to the caller */
};

/* One past the last job of the chunk that starts at job j0: the whole jobs that fit both an output slot (STAGE_OUT
 * decoded bytes) and an input slot (STAGE_IN compressed bytes).  j0 itself when job j0 alone does not fit. */
static uint32_t staged_chunk_end(const zxc_b200_job_t* jobs, uint32_t n_jobs, uint32_t j0) {
    uint32_t j1 = j0;
    uint64_t out = 0, in = 0;
    while (j1 < n_jobs && out + jobs[j1].dst_cap <= STAGE_OUT && in + jobs[j1].src_len <= STAGE_IN) {
        out += jobs[j1].dst_cap;
        in += jobs[j1].src_len;
        j1++;
    }
    return j1;
}

extern "C" int zxg_decode_staged(zxg_ctx* c, const uint8_t* h_src, zxg_fetch_fn fetch, void* fetch_ctx, uint64_t src_lo,
                                 uint64_t src_hi, uint8_t* h_dst, uint64_t clip_lo, uint64_t clip_hi,
                                 const zxc_b200_job_t* h_jobs, uint32_t n_jobs, int32_t* h_status, const void* h_dict,
                                 uint32_t dict_size, const void* h_dict_huf, uint32_t block_size, int verify_checksums) {
    if (n_jobs == 0) return ZXC_OK;
    int rc = staged_ready(c);
    if (rc != ZXC_OK) return rc;
    const uint64_t produced = h_jobs[n_jobs - 1].dst_off + h_jobs[n_jobs - 1].dst_cap;
    u8* d_in = (u8*)zxg_buffer(c, ZXG_BUF_IN, (size_t)(src_hi - src_lo) + 16);
    u8* d_out = (u8*)zxg_buffer(c, ZXG_BUF_OUT, (size_t)produced + 16);
    zxc_b200_job_t* d_jobs = (zxc_b200_job_t*)zxg_buffer(c, ZXG_BUF_JOBS, (size_t)n_jobs * sizeof(zxc_b200_job_t));
    i32* d_status = (i32*)zxg_buffer(c, ZXG_BUF_STATUS, (size_t)n_jobs * sizeof(i32));
    /* a chunk holds at most STAGE_OUT / (smallest decoded block) jobs; every slot decodes on its own stream with its
     * own scratch region and work counters, so up to STAGE_SLOTS chunk launches are resident together */
    uint32_t chunk_jobs_max = 1;
    for (uint32_t j = 0; j < n_jobs;) {
        const uint32_t j1 = staged_chunk_end(h_jobs, n_jobs, j);
        if (j1 == j) break;
        if (j1 - j > chunk_jobs_max) chunk_jobs_max = j1 - j;
        j = j1;
    }
    const size_t scratch_size = (launch_scratch_bytes(chunk_jobs_max, block_size) + 255) & ~(size_t)255;
    u8* d_scratch = (u8*)zxg_buffer(c, ZXG_BUF_SCRATCH, scratch_size * STAGE_SLOTS);
    if (!d_in || !d_out || !d_jobs || !d_status || !d_scratch) return ZXC_ERROR_MEMORY;
    u8 *d_dict, *d_huf;
    rc = upload_dict(c, h_dict, dict_size, h_dict_huf, &d_dict, &d_huf);
    if (rc != ZXC_OK) return rc;
    if (cudaMemcpyAsync(d_jobs, h_jobs, (size_t)n_jobs * sizeof(zxc_b200_job_t), cudaMemcpyHostToDevice, c->stream) != cudaSuccess)
        return ZXC_B200_ERROR_CUDA;
    cudaStreamSynchronize(c->stream); /* h_jobs may be pageable: do not let the caller free it under the copy */

    staged_chunk ring[STAGE_SLOTS];
    uint32_t j0 = 0, issued = 0, drained = 0;
    copy_pool* drain_job = NULL; /* the drain in flight on the second pool ... */
    int drain_slot = -1;         /* ... and the output slot it is reading */
    while (rc == ZXC_OK && (drained < issued || j0 < n_jobs)) {
        /* one slot is always left to the drain in flight, so filling the next chunk never waits for it */
        if (j0 < n_jobs && issued - drained < STAGE_SLOTS - 1) { /* a slot is free: stage and queue the next chunk */
            const int slot = (int)(issued % STAGE_SLOTS);
            staged_chunk ch;
            ch.j0 = j0;
            const uint32_t j1 = staged_chunk_end(h_jobs, n_jobs, j0);
            if (j1 == j0) { /* a single block larger than a stage: cannot happen with <= 2 MiB blocks */
                rc = ZXC_ERROR_MEMORY;
                break;
            }
            ch.j1 = j1;
            ch.s0 = h_jobs[j0].src_off;
            ch.s1 = h_jobs[j1 - 1].src_off + h_jobs[j1 - 1].src_len;
            const uint64_t o0 = h_jobs[j0].dst_off, o1 = h_jobs[j1 - 1].dst_off + h_jobs[j1 - 1].dst_cap;
            ch.c0 = o0 > clip_lo ? o0 : clip_lo;
            ch.c1 = o1 < clip_hi ? o1 : clip_hi;
            if (ch.c1 < ch.c0) ch.c1 = ch.c0;
            if (drain_job && drain_slot == slot) { /* this chunk's D2H will overwrite what the drain is still reading */
                pool_copy_end(drain_job);
                drain_job = NULL;
            }
            cudaEventSynchronize(c->st_ev_in[slot]); /* the slot's previous H2D has left the bounce buffer */
            u8* pin = (u8*)c->st_in[slot].p;
            if (fetch) {
                rc = fetch(fetch_ctx, pin, (size_t)(ch.s1 - ch.s0), ch.s0);
                if (rc != ZXC_OK) break;
            } else {
                pool_memcpy(c->device, pin, h_src + ch.s0, (size_t)(ch.s1 - ch.s0));
            }
            if (cudaMemcpyAsync(d_in + (ch.s0 - src_lo), pin, (size_t)(ch.s1 - ch.s0), cudaMemcpyHostToDevice, c->s_h2d) != cudaSuccess) {
                rc = ZXC_B200_ERROR_CUDA;
                break;
            }
            cudaEventRecord(c->st_ev_in[slot], c->s_h2d);
            cudaStreamWaitEvent(c->s_dec[slot], c->st_ev_in[slot], 0);
            rc = launch_decode(d_in - src_lo, d_out, d_jobs + j0, j1 - j0, d_status + j0, d_dict, dict_size, d_huf,
                               d_scratch + (size_t)slot * scratch_size, scratch_size, block_size, verify_checksums,
                               c->counter + 4 * slot, c->s_dec[slot], 0);
            if (rc != ZXC_OK) break;
            cudaEventRecord(c->st_ev_dec[slot], c->s_dec[slot]);
            cudaStreamWaitEvent(c->s_d2h, c->st_ev_dec[slot], 0);
            if (ch.c1 > ch.c0 &&
                cudaMemcpyAsync(c->st_out[slot].p, d_out + ch.c0, (size_t)(ch.c1 - ch.c0), cudaMemcpyDeviceToHost, c->s_d2h) != cudaSuccess) {
                rc = ZXC_B200_ERROR_CUDA;
                break;
            }
            cudaEventRecord(c->st_ev_out[slot], c->s_d2h);
            ring[slot] = ch;
            j0 = j1;
            issued++;
            if (j0 < n_jobs && issued - drained < STAGE_SLOTS - 1) continue; /* fill the pipeline before draining */
        }
        /* hand the oldest finished chunk to the caller while the GPU works on the younger ones */
        const int ds = (int)(drained % STAGE_SLOTS);
        if (cudaEventSynchronize(c->st_ev_out[ds]) != cudaSuccess) {
            rc = ZXC_B200_ERROR_CUDA;
            break;
        }
        const staged_chunk& dc = ring[ds];
        pool_copy_end(drain_job); /* one drain at a time; the previous one overlapped the fill above */
        drain_job = NULL;
        if (dc.c1 > dc.c0) drain_job = pool_copy_begin(c->device, h_dst + (dc.c0 - clip_lo), c->st_out[ds].p, (size_t)(dc.c1 - dc.c0));
        drain_slot = ds;
        drained++;
    }
    pool_copy_end(drain_job);
    cudaError_t e0 = cudaSuccess;
    for (int i = 0; i < STAGE_SLOTS; i++) {
        const cudaError_t e = cudaStreamSynchronize(c->s_dec[i]);
        if (e != cudaSuccess) e0 = e;
    }
    if (rc == ZXC_OK &&
        cudaMemcpyAsync(h_status, d_status, (size_t)n_jobs * sizeof(i32), cudaMemcpyDeviceToHost, c->stream) != cudaSuccess)
        rc = ZXC_B200_ERROR_CUDA;
    const cudaError_t e1 = cudaStreamSynchronize(c->stream);
    const cudaError_t e2 = cudaStreamSynchronize(c->s_d2h);
    const cudaError_t e3 = cudaStreamSynchronize(c->s_h2d);
    if (e0 != cudaSuccess || e1 != cudaSuccess || e2 != cudaSuccess || e3 != cudaSuccess) {
        fprintf(stderr, "libzxc (CUDA build): staged decode failed: %s\n", cudaGetErrorString(cudaGetLastError()));
        return ZXC_B200_ERROR_CUDA;
    }
    return rc;
}

/* ------------------------------------------------------------------------- */
/* frame body encode: blocks -> per-block slots -> compacted body             */
/* ------------------------------------------------------------------------- */
static u32 enc_staging_stride(u32 bs) { return ((bs + 8u + 68u + 4u) + 255u) & ~255u; }

/* dictionary region of an encode: [dict (padded)] [seeded head 128 KB] [seeded chain 128 KB] [256 literal lengths];
 * a prepared dictionary's region holds two head / chain pairs (zxc_seed_kernel depends on the level only through
 * hash5 = level >= 3): enc_dict_bytes(dict_size, 2) */
static const size_t ENC_SEED_PAIR = (size_t)ENC_HASH_SIZE * 4 + (size_t)ENC_WINDOW * 2;
static size_t enc_dict_pad(u32 dict_size) { return ((size_t)dict_size + 16 + 255) & ~(size_t)255; }
static size_t enc_dict_bytes(u32 dict_size, u32 pairs = 1) {
    return enc_dict_pad(dict_size) + pairs * ENC_SEED_PAIR + 256;
}

/* warps of the full resident encode grid for n_blocks blocks (a multiple of ENC_WARPS_PER_CTA) */
static u32 enc_full_warps(u32 n_blocks) {
    const u32 ctas_needed = (n_blocks + ENC_WARPS_PER_CTA - 1) / ENC_WARPS_PER_CTA;
    const u32 resident = (u32)(g_sm_count > 0 ? g_sm_count : 132) * ENC_CTAS_PER_SM;
    return (ctas_needed < resident ? ctas_needed : resident) * ENC_WARPS_PER_CTA;
}

/* One block encode on stream `st` with the given device buffers: d_src is 16-byte aligned with 64 zero bytes behind
 * src_size, d_scratch holds `warps` per-warp slots of enc_layout(block_size, level).total bytes, d_dict (when
 * dict_size) holds enc_dict_bytes(dict_size).  The host dictionary (<= ZXC_DICT_SIZE_MAX bytes) and literal lengths
 * are copied in here, unless a prepared dictionary dd is given.  Launches the seed kernel (host dictionary only) and
 * the encode kernel: `warps` warps, in CTAs of
 * ENC_WARPS_PER_CTA when there are that many, else one CTA of `warps` warps (the kernel indexes its scratch by
 * global warp and claims blocks through *counter, so any warp count gives the same output). */
struct EncLaunch {
    const u8* d_src;
    uint64_t src_size;
    u32 block_size, n_blocks;
    int level, checksum;
    u8* d_stage;
    u32* d_sizes;
    u8* d_scratch;
    u32 warps;
    unsigned long long* counter;
    u8* d_dict;
    const void* h_dict;
    u32 dict_size;
    const uint8_t* h_dict_huf_lens;
    const zxg_ddict_t* dd; /* or a prepared dictionary (h_dict NULL) */
};
/* Builds the dictionary region of an encode at d_dict (enc_dict_bytes(dict_size, pairs) bytes): the host dictionary,
 * read through a pageable copy (host_bounce) so the call has read it when it returns, and the literal lengths when
 * given, copied in; head / chain pair k seeded by zxc_seed_kernel for levels[k] (one launch each). */
static void* host_bounce(const void* p, size_t n, size_t bytes);
static int enc_build_dict(u8* d_dict, const void* h_dict, u32 dict_size, const int* levels, u32 pairs,
                          const uint8_t* h_dict_huf_lens, cudaStream_t st) {
    void* bd = host_bounce(h_dict, dict_size, dict_size);
    if (!bd) return ZXC_ERROR_MEMORY;
    const size_t dpad = enc_dict_pad(dict_size);
    const bool ok = cudaMemsetAsync(d_dict, 0, enc_dict_bytes(dict_size, pairs), st) == cudaSuccess &&
                    cudaMemcpyAsync(d_dict, bd, dict_size, cudaMemcpyHostToDevice, st) == cudaSuccess;
    free(bd);
    if (!ok) return ZXC_B200_ERROR_CUDA;
    if (h_dict_huf_lens && /* the shared literal table, one length per byte */
        cudaMemcpyAsync(d_dict + dpad + pairs * ENC_SEED_PAIR, h_dict_huf_lens, 256, cudaMemcpyHostToDevice, st) !=
            cudaSuccess)
        return ZXC_B200_ERROR_CUDA;
    for (u32 k = 0; k < pairs; k++) {
        u8* pair = d_dict + dpad + k * ENC_SEED_PAIR;
        zxc_seed_kernel<<<1, 32, 0, st>>>(d_dict, dict_size, (u32)levels[k], (u32*)pair,
                                          (unsigned short*)(pair + (size_t)ENC_HASH_SIZE * 4));
        __atomic_add_fetch(&g_launches, 1, __ATOMIC_RELAXED);
    }
    return ZXC_OK;
}

/* Points P's dictionary fields at a region laid out by enc_build_dict: head / chain pair `pair`, the literal lengths
 * when has_lens and the level reads them (6-7). */
static void enc_point_dict(EncodeParams& P, const u8* d_dict, u32 dict_size, u32 pairs, u32 pair, bool has_lens,
                           int level) {
    const u8* seeds = d_dict + enc_dict_pad(dict_size);
    P.dict = d_dict;
    P.seed_head = (const u32*)(seeds + pair * ENC_SEED_PAIR);
    P.seed_chain = (const unsigned short*)(seeds + pair * ENC_SEED_PAIR + (size_t)ENC_HASH_SIZE * 4);
    if (has_lens && level >= 6) P.dict_huf_lens = seeds + pairs * ENC_SEED_PAIR;
}

/* The dictionary of an encode at this level, into P: the host dictionary staged into the region at d_dict (one
 * seeding launch), or the prepared dictionary dd used where it lies (no launch); with_lens: dd's literal lengths apply
 * (the block API attaches none). */
static int enc_stage_dict(EncodeParams& P, u8* d_dict, const void* h_dict, u32 dict_size, int level,
                          const uint8_t* h_dict_huf_lens, const zxg_ddict_t* dd, bool with_lens, cudaStream_t st) {
    if (dd) {
        enc_point_dict(P, (const u8*)dd->enc, dd->dict_size, 2, level >= 3 ? 1 : 0, with_lens && dd->enc_lens, level);
        return ZXC_OK;
    }
    const uint8_t* lens = level >= 6 ? h_dict_huf_lens : NULL;
    const int rc = enc_build_dict(d_dict, h_dict, dict_size, &level, 1, lens, st);
    if (rc == ZXC_OK) enc_point_dict(P, d_dict, dict_size, 1, 0, lens != NULL, level);
    return rc;
}

/* The encode kernel on E's blocks with the dictionary fields already in P (staged once for several launches) */
static int launch_encode_staged(EncodeParams P, const EncLaunch& E, cudaStream_t st) {
    P.src = E.d_src;
    P.staging = E.d_stage;
    P.out_size = E.d_sizes;
    P.scratch = E.d_scratch;
    P.counter = E.counter;
    P.src_size = E.src_size;
    P.scratch_stride = enc_layout(E.block_size, E.level).total;
    P.block_size = E.block_size;
    P.n_blocks = E.n_blocks;
    P.staging_stride = enc_staging_stride(E.block_size);
    P.level = (u32)E.level;
    P.checksum = E.checksum ? 1u : 0u;
    P.dict_size = P.dict ? (E.dd ? E.dd->dict_size : E.dict_size) : 0;
    if (cudaMemsetAsync(E.counter, 0, sizeof(unsigned long long), st) != cudaSuccess) return ZXC_B200_ERROR_CUDA;
    const u32 grid = E.warps >= ENC_WARPS_PER_CTA ? E.warps / ENC_WARPS_PER_CTA : 1u;
    const u32 threads = E.warps >= ENC_WARPS_PER_CTA ? ENC_CTA_THREADS : 32u * E.warps;
    if (E.level >= 6) zxc_encode_kernel<true><<<grid, threads, 0, st>>>(P);
    else zxc_encode_kernel<false><<<grid, threads, 0, st>>>(P);
    __atomic_add_fetch(&g_launches, 1, __ATOMIC_RELAXED);
    return cudaGetLastError() == cudaSuccess ? ZXC_OK : ZXC_B200_ERROR_CUDA;
}

static EncodeParams enc_no_dict(void) {
    EncodeParams P;
    P.dict = NULL;
    P.seed_head = NULL;
    P.seed_chain = NULL;
    P.dict_huf_lens = NULL;
    return P;
}

static int launch_encode(const EncLaunch& E, cudaStream_t st) {
    EncodeParams P = enc_no_dict();
    if (E.dd || (E.h_dict && E.dict_size)) {
        const int rc = enc_stage_dict(P, E.d_dict, E.h_dict, E.dict_size, E.level, E.h_dict_huf_lens, E.dd, true, st);
        if (rc != ZXC_OK) return rc;
    }
    return launch_encode_staged(P, E, st);
}

/* gather the staging slots to out + dst_off[j] */
static void launch_compact(const u8* d_stage, u32 sstride, const unsigned long long* d_offs, const u32* d_sizes,
                           u8* out, u32 n_blocks, cudaStream_t st) {
    const u32 cmax = (u32)(g_sm_count > 0 ? g_sm_count : 132) * 8u;
    const u32 cgrid = (n_blocks + 7) / 8 < cmax ? (n_blocks + 7) / 8 : cmax;
    zxc_compact_kernel<<<cgrid, 256, 0, st>>>(d_stage, sstride, d_offs, d_sizes, out, n_blocks);
    __atomic_add_fetch(&g_launches, 1, __ATOMIC_RELAXED);
}

/* Encodes src into the frame BODY (all data blocks back to back) in h_body.  h_sizes receives
 * n_blocks on-disk block sizes.  Returns ZXC_OK, or ZXC_ERROR_DST_TOO_SMALL when the body does
 * not fit body_cap (then *body_size holds the size that would have been needed). */
extern "C" int zxg_encode_body(zxg_ctx* c, const uint8_t* h_src, uint64_t src_size, uint32_t block_size, int level,
                               int checksum, uint32_t n_blocks, uint8_t* h_body, uint64_t body_cap,
                               uint32_t* h_sizes, uint64_t* body_size, const void* h_dict, uint32_t dict_size,
                               const uint8_t* h_dict_huf_lens) {
    *body_size = 0;
    if (n_blocks == 0) return ZXC_OK;
    const u32 sstride = enc_staging_stride(block_size);
    const size_t wstride = enc_layout(block_size, level).total;
    const u32 warps = enc_full_warps(n_blocks);
    u8* d_src = (u8*)zxg_buffer(c, ZXG_BUF_IN, (size_t)src_size + 64);
    u8* d_stage = (u8*)zxg_buffer(c, ZXG_BUF_OUT, (size_t)n_blocks * sstride);
    u8* d_scratch = (u8*)zxg_buffer(c, ZXG_BUF_SCRATCH, (size_t)warps * wstride);
    u32* d_sizes = (u32*)zxg_buffer(c, ZXG_BUF_STATUS, (size_t)n_blocks * 4);
    unsigned long long* d_offs = (unsigned long long*)zxg_buffer(c, ZXG_BUF_JOBS, (size_t)n_blocks * 8);
    if (!d_src || !d_stage || !d_scratch || !d_sizes || !d_offs) return ZXC_ERROR_MEMORY;
    int rc = zxg_h2d(c, d_src, h_src, (size_t)src_size);
    if (rc != ZXC_OK) return rc;
    if (cudaMemsetAsync(d_src + src_size, 0, 64, c->stream) != cudaSuccess) return ZXC_B200_ERROR_CUDA;
    u8* d_dict = NULL;
    if (h_dict && dict_size) {
        d_dict = (u8*)zxg_buffer(c, ZXG_BUF_DICT, enc_dict_bytes(dict_size));
        if (!d_dict) return ZXC_ERROR_MEMORY;
    }
    const EncLaunch E = {d_src, src_size, block_size, n_blocks, level, checksum, d_stage, d_sizes, d_scratch, warps,
                         c->counter, d_dict, h_dict, dict_size, h_dict_huf_lens, NULL};
    rc = launch_encode(E, c->stream);
    if (rc != ZXC_OK) return rc;
    if (cudaMemcpyAsync(h_sizes, d_sizes, (size_t)n_blocks * 4, cudaMemcpyDeviceToHost, c->stream) != cudaSuccess ||
        cudaStreamSynchronize(c->stream) != cudaSuccess) {
        fprintf(stderr, "libzxc (CUDA build): encode kernel failed: %s\n", cudaGetErrorString(cudaGetLastError()));
        return ZXC_B200_ERROR_CUDA;
    }
    unsigned long long* h_offs = (unsigned long long*)malloc((size_t)n_blocks * 8);
    if (!h_offs) return ZXC_ERROR_MEMORY;
    uint64_t acc = 0;
    for (u32 i = 0; i < n_blocks; i++) {
        h_offs[i] = acc;
        acc += h_sizes[i];
    }
    *body_size = acc;
    if (acc > body_cap) {
        free(h_offs);
        return ZXC_ERROR_DST_TOO_SMALL;
    }
    /* the input buffer is no longer needed: reuse it for the compacted body when it is big enough */
    u8* d_body = (u8*)zxg_buffer(c, ZXG_BUF_AUX, (size_t)acc + 16);
    rc = d_body ? zxg_h2d(c, d_offs, h_offs, (size_t)n_blocks * 8) : ZXC_ERROR_MEMORY;
    if (rc == ZXC_OK) {
        launch_compact(d_stage, sstride, d_offs, d_sizes, d_body, n_blocks, c->stream);
        rc = zxg_d2h(c, h_body, d_body, (size_t)acc);
        if (rc == ZXC_OK) rc = zxg_sync(c);
    }
    free(h_offs);
    return rc;
}

/* ------------------------------------------------------------------------- */
/* device-to-device compress (zxc_b200_compress_device): the encode above,   */
/* then the frame assembled on the device (zxc_assemble.cuh)                 */
/* ------------------------------------------------------------------------- */
/* Scratch layout, from the caller's base rounded up to 256 bytes (every region 256-aligned):
 *   AsmState (256) | input copy + 64 zero bytes | dictionary region (with a dictionary) | staging slots |
 *   sizes (u32 per block) | body offsets (u64 per block) | tile sums (u64 per ASM_TILE blocks) | per-warp encode slots
 * The caller's input is copied into the scratch (device to device) so the encode kernel gets the aligned, padded
 * input it assumes (EncodeParams::src) whatever the caller's alignment and allocation end. */
/* A copy of n host bytes (of a buffer of `bytes`) in fresh pageable memory.  cudaMemcpyAsync from pageable memory
 * returns only once it has read the source (it stages it for the DMA), while from page-locked memory it returns before
 * the copy runs: the device-to-device calls promise to have read the caller's dictionary when they return, so a
 * caller may reuse even a pinned one at once.  NULL on allocation failure; the caller frees it after the copy call. */
static void* host_bounce(const void* p, size_t n, size_t bytes) {
    void* b = malloc(bytes);
    if (b) memcpy(b, p, n);
    return b;
}

struct DevEncLayout {
    size_t in, dict, stage, sizes, offs, tiles, warps, fixed; /* fixed: bytes before the first warp slot + base slack */
    size_t wstride;
};
static size_t r256(size_t v) { return (v + 255) & ~(size_t)255; }
static DevEncLayout dev_enc_layout(uint64_t src_size, u32 block_size, u32 n_blocks, int level, u32 dict_size) {
    DevEncLayout L;
    size_t o = 256;
    L.in = o;
    o += r256((size_t)src_size + 64);
    L.dict = o;
    if (dict_size) o += r256(enc_dict_bytes(dict_size));
    L.stage = o;
    o += (size_t)n_blocks * enc_staging_stride(block_size);
    L.sizes = o;
    o += r256((size_t)n_blocks * 4);
    L.offs = o;
    o += r256((size_t)n_blocks * 8);
    L.tiles = o;
    o += r256(((size_t)n_blocks + ASM_TILE - 1) / ASM_TILE * 8);
    L.warps = o;
    L.fixed = o + 256;
    L.wstride = enc_layout(block_size, level).total;
    return L;
}

extern "C" size_t zxg_encode_scratch_bytes(uint64_t src_size, uint32_t block_size, int level, uint32_t n_blocks,
                                           uint32_t dict_size) {
    if (zxg_init() != ZXC_OK) return 0;
    const DevEncLayout L = dev_enc_layout(src_size, block_size, n_blocks, level, dict_size);
    return L.fixed + (size_t)(n_blocks ? enc_full_warps(n_blocks) : 1u) * L.wstride;
}

extern "C" int zxg_compress_device(const void* d_src, uint64_t src_size, void* d_dst, uint32_t block_size, int level,
                                   int checksum, uint32_t n_blocks, const void* h_dict, uint32_t dict_size,
                                   const uint8_t* h_dict_huf_lens, const zxg_ddict_t* dd, const zxg_frame_bytes_t* fb,
                                   void* d_scratch, size_t scratch_size, int64_t* d_result, zxc_b200_job_t* d_jobs,
                                   void* stream) {
    const int irc = zxg_init();
    if (irc != ZXC_OK) return irc;
    const DevEncLayout L = dev_enc_layout(src_size, block_size, n_blocks, level, dict_size);
    if (scratch_size < L.fixed + L.wstride) return ZXC_ERROR_MEMORY;
    const size_t fit = (scratch_size - L.fixed) / L.wstride;
    const u32 full = n_blocks ? enc_full_warps(n_blocks) : 1u;
    const u32 warps = fit < full ? (u32)fit : full;
    cudaStream_t st = (cudaStream_t)stream;
    u8* base = (u8*)(((uintptr_t)d_scratch + 255) & ~(uintptr_t)255);
    AsmState* state = (AsmState*)base;
    u8* d_dst8 = (u8*)d_dst;
    AsmFrame F;
    memcpy(F.header, fb->header, 16);
    memcpy(F.eof, fb->eof, 8);
    memcpy(F.sek, fb->sek, 8);
    memcpy(F.footer, fb->footer, 12);
    F.src_size = src_size;
    F.dst_capacity = fb->dst_capacity;
    F.fixed = fb->fixed;
    F.n_blocks = n_blocks;
    F.block_size = block_size;
    F.staging_stride = enc_staging_stride(block_size);
    F.checksum = checksum ? 1u : 0u;
    F.seekable = fb->seekable ? 1u : 0u;
    if (n_blocks) {
        u8* d_in = base + L.in;
        u8* d_stage = base + L.stage;
        u32* d_sizes = (u32*)(base + L.sizes);
        unsigned long long* d_offs = (unsigned long long*)(base + L.offs);
        unsigned long long* d_tiles = (unsigned long long*)(base + L.tiles);
        const u32 n_tiles = (u32)(((uint64_t)n_blocks + ASM_TILE - 1) / ASM_TILE);
        if (cudaMemcpyAsync(d_in, d_src, (size_t)src_size, cudaMemcpyDeviceToDevice, st) != cudaSuccess ||
            cudaMemsetAsync(d_in + src_size, 0, 64, st) != cudaSuccess)
            return ZXC_B200_ERROR_CUDA;
        const EncLaunch E = {d_in, src_size, block_size, n_blocks, level, checksum, d_stage, d_sizes, base + L.warps,
                             warps, &state->counter, base + L.dict, h_dict, dict_size, h_dict_huf_lens, dd};
        const int rc = launch_encode(E, st);
        if (rc != ZXC_OK) return rc;
        zxc_asm_tile_sums<<<n_tiles, ASM_THREADS, 0, st>>>(d_sizes, n_blocks, d_tiles);
        zxc_asm_scan_tiles<<<1, ASM_SCAN_THREADS, 0, st>>>(d_tiles, n_tiles, state, F);
        zxc_asm_blocks<<<n_tiles, ASM_THREADS, 0, st>>>(d_sizes, d_stage, d_tiles, d_offs, state, d_jobs, d_dst8, F);
        __atomic_add_fetch(&g_launches, 3, __ATOMIC_RELAXED);
        launch_compact(d_stage, F.staging_stride, d_offs, d_sizes, d_dst8 + 16 /* file header */, n_blocks, st);
    }
    zxc_asm_finish<<<1, 1, 0, st>>>(d_dst8, state, F, (long long*)d_result);
    __atomic_add_fetch(&g_launches, 1, __ATOMIC_RELAXED);
    return cudaGetLastError() == cudaSuccess ? ZXC_OK : ZXC_B200_ERROR_CUDA;
}

/* ------------------------------------------------------------------------- */
/* device buffer to a frame in page-locked host memory, window by window     */
/* (zxc_b200_compress_device_to_host: kernels in zxc_c2host.cuh)             */
/* ------------------------------------------------------------------------- */
/* Scratch layout, from the caller's base rounded up to 256 bytes (every region 256-aligned), for windows of wb blocks:
 *   C2hState (256) | input copy of one window + 64 zero bytes | dictionary region (with a host dictionary) |
 *   staging slots (wb) | sizes (u32 x wb) | body offsets (u64 x wb) | tile sums (u64 per ASM_TILE of wb) |
 *   SEK entries (u32 x n, seekable only) | per-warp encode slots */
static DevEncLayout c2h_layout(u64 W, u32 block_size, u32 n_blocks, int level, u32 dict_size, int seekable,
                               size_t* sek) {
    const u32 wb = (u32)(W / block_size);
    DevEncLayout L = dev_enc_layout(W, block_size, wb, level, dict_size);
    *sek = L.warps;
    if (seekable) L.warps += r256((size_t)n_blocks * 4);
    L.fixed = L.warps + 256;
    return L;
}

/* window rounded up to whole blocks, capped at the input rounded up to a block, at least one block */
static u64 c2h_window(uint64_t src_size, uint64_t window, u32 block_size) {
    const u64 cap = (src_size + block_size - 1) / block_size * block_size;
    u64 W = window / block_size + (window % block_size != 0);
    W = W > (cap / block_size) ? cap : W * block_size;
    return W < block_size ? block_size : W;
}

extern "C" size_t zxg_c2h_scratch_bytes(uint64_t src_size, uint64_t window, uint32_t block_size, int level,
                                        uint32_t n_blocks, uint32_t dict_size, int seekable) {
    if (zxg_init() != ZXC_OK) return 0;
    const u64 W = c2h_window(src_size, window, block_size);
    size_t sek;
    const DevEncLayout L = c2h_layout(W, block_size, n_blocks, level, dict_size, seekable, &sek);
    return L.fixed + (size_t)enc_full_warps((u32)(W / block_size)) * L.wstride;
}

extern "C" int zxg_compress_device_to_host(const void* d_src, uint64_t src_size, void* h_mapped, uint64_t window,
                                           uint32_t block_size, int level, int checksum, uint32_t n_blocks,
                                           const void* h_dict, uint32_t dict_size, const uint8_t* h_dict_huf_lens,
                                           const zxg_ddict_t* dd, const zxg_frame_bytes_t* fb, void* d_scratch,
                                           size_t scratch_size, int64_t* d_result, void* stream) {
    const int irc = zxg_init();
    if (irc != ZXC_OK) return irc;
    const u64 W = c2h_window(src_size, window, block_size);
    const u32 wb = (u32)(W / block_size);
    size_t sek_off;
    const DevEncLayout L = c2h_layout(W, block_size, n_blocks, level, dict_size, fb->seekable, &sek_off);
    if (scratch_size < L.fixed + L.wstride) return ZXC_ERROR_MEMORY;
    const size_t fit = (scratch_size - L.fixed) / L.wstride;
    const u32 full = enc_full_warps(wb);
    const u32 warps = fit < full ? (u32)fit : full;
    cudaStream_t st = (cudaStream_t)stream;
    u8* base = (u8*)(((uintptr_t)d_scratch + 255) & ~(uintptr_t)255);
    C2hState* state = (C2hState*)base;
    u8* hd = (u8*)h_mapped;
    u32* d_sek = fb->seekable ? (u32*)(base + sek_off) : NULL;
    const u32 sstride = enc_staging_stride(block_size);
    const u32 gmax = (u32)(g_sm_count > 0 ? g_sm_count : 132) * 8u;
    if (cudaMemsetAsync(state, 0, sizeof(C2hState), st) != cudaSuccess) return ZXC_B200_ERROR_CUDA;
    EncodeParams P = enc_no_dict();
    if (n_blocks && (dd || (h_dict && dict_size))) { /* staged once for every round */
        const int rc = enc_stage_dict(P, base + L.dict, h_dict, dict_size, level, h_dict_huf_lens, dd, true, st);
        if (rc != ZXC_OK) return rc;
    }
    C2hHeader H;
    memcpy(H.b, fb->header, 16);
    u32 rounds = 0;
    for (u64 s0 = 0; s0 < src_size; s0 += W, rounds++) {
        const u64 len = src_size - s0 < W ? src_size - s0 : W;
        const u32 wn = (u32)((len + block_size - 1) / block_size);
        const u32 j0 = (u32)(s0 / block_size);
        u8* d_in = base + L.in;
        u8* d_stage = base + L.stage;
        u32* d_sizes = (u32*)(base + L.sizes);
        unsigned long long* d_offs = (unsigned long long*)(base + L.offs);
        unsigned long long* d_tiles = (unsigned long long*)(base + L.tiles);
        const u32 n_tiles = (wn + ASM_TILE - 1) / ASM_TILE;
        if (cudaMemcpyAsync(d_in, (const u8*)d_src + s0, (size_t)len, cudaMemcpyDeviceToDevice, st) != cudaSuccess ||
            cudaMemsetAsync(d_in + len, 0, 64, st) != cudaSuccess)
            return ZXC_B200_ERROR_CUDA;
        const EncLaunch E = {d_in, len, block_size, wn, level, checksum, d_stage, d_sizes, base + L.warps,
                             warps, &state->counter, base + L.dict, h_dict, dict_size, h_dict_huf_lens, dd};
        const int rc = launch_encode_staged(P, E, st);
        if (rc != ZXC_OK) return rc;
        const u64 chunks = ((u64)wn * sstride + 15) / 16 + 1;
        const u32 wgrid = (u32)((chunks + C2H_THREADS - 1) / C2H_THREADS < gmax ? (chunks + C2H_THREADS - 1) / C2H_THREADS
                                                                                 : gmax);
        zxc_asm_tile_sums<<<n_tiles, ASM_THREADS, 0, st>>>(d_sizes, wn, d_tiles);
        zxc_c2h_scan<<<1, ASM_SCAN_THREADS, 0, st>>>(d_tiles, n_tiles, state, fb->fixed, fb->dst_capacity);
        zxc_c2h_blocks<<<n_tiles, ASM_THREADS, 0, st>>>(d_sizes, d_stage, d_tiles, d_offs, state, d_sek, wn, j0,
                                                        n_blocks, sstride, checksum ? 1u : 0u);
        zxc_c2h_write<<<wgrid, C2H_THREADS, 0, st>>>(hd, d_stage, sstride, d_offs, d_sizes, wn, state, H, rounds & 1u);
        __atomic_add_fetch(&g_launches, 4, __ATOMIC_RELAXED);
        if (cudaGetLastError() != cudaSuccess) return ZXC_B200_ERROR_CUDA;
    }
    C2hFinish F;
    memcpy(F.header, fb->header, 16);
    memcpy(F.eof, fb->eof, 8);
    memcpy(F.sek, fb->sek, 8);
    memcpy(F.footer, fb->footer, 12);
    F.dst_capacity = fb->dst_capacity;
    F.fixed = fb->fixed;
    F.n_blocks = n_blocks;
    F.checksum = checksum ? 1u : 0u;
    F.seekable = fb->seekable ? 1u : 0u;
    F.parity = rounds & 1u;
    const u64 tchunks = (fb->fixed + 31) / 16 + 2; /* the trailer, the carried tail and chunk 0 */
    const u32 fgrid = (u32)((tchunks + C2H_THREADS - 1) / C2H_THREADS < gmax ? (tchunks + C2H_THREADS - 1) / C2H_THREADS
                                                                              : gmax);
    zxc_c2h_finish<<<fgrid, C2H_THREADS, 0, st>>>(hd, (const u8*)d_sek, state, F, (long long*)d_result);
    __atomic_add_fetch(&g_launches, 1, __ATOMIC_RELAXED);
    return cudaGetLastError() == cudaSuccess ? ZXC_OK : ZXC_B200_ERROR_CUDA;
}

/* ------------------------------------------------------------------------- */
/* many device-resident buffers compressed in one call                       */
/* (zxc_b200_compress_device_batch: kernels in zxc_cbatch.cuh)               */
/* ------------------------------------------------------------------------- */
/* Scratch layout, from the caller's base rounded up to 256 bytes (every region 256-aligned):
 *   CBatchState | frames (n x CBatchFrame) | first blocks (n x u64) | frame tile sums (2 per tile) | dictionary region
 *   (with a dictionary) | offsets (nb_max x u64) | sizes (nb_max x u32) | block tile sums | room: the pool (256 x
 *   pool_units bytes), then one encode slot
 * Everything but the pool follows from (n, options, pool_units): nb_max = max(1, pool / (staging_stride + 256)) is the
 * most blocks a pool can hold (every block's share, with its frame's input, is at least that).  The call takes the
 * largest pool whose layout fits the scratch, and launches W = min(resident grid, nb_max) encode warps (whole CTAs
 * from ENC_WARPS_PER_CTA up); those whose slot, counted down from the room's end, reaches the pool's used part exit. */
struct CBatchLayout {
    size_t frames, first, ftiles, dict, offs, sizes, btiles, pool, total, wstride;
    u32 W, nb_max, stride;
    u64 pool_units;
};
#define CB_FRAMES_MAX (1u << 30)

static void cb_layout(u32 n, u32 bs, int level, u32 dict_size, u64 pool_units, CBatchLayout* L) {
    const size_t n_tiles = ((size_t)n + ASM_TILE - 1) / ASM_TILE;
    L->stride = enc_staging_stride(bs);
    L->wstride = enc_layout(bs, level).total;
    const u64 nb = pool_units * 256 / ((u64)L->stride + 256);
    L->nb_max = nb ? (u32)nb : 1u;
    const u32 resident = (u32)(g_sm_count > 0 ? g_sm_count : 132) * ENC_CTAS_PER_SM * ENC_WARPS_PER_CTA;
    u32 W = L->nb_max < resident ? L->nb_max : resident;
    if (W >= ENC_WARPS_PER_CTA) W -= W % ENC_WARPS_PER_CTA;
    L->W = W;
    L->pool_units = pool_units;
    size_t o = CB_STATE_BYTES;
    L->frames = o;
    o += r256((size_t)n * sizeof(CBatchFrame));
    L->first = o;
    o += r256((size_t)n * 8);
    L->ftiles = o;
    o += r256(n_tiles * 16);
    L->dict = o;
    if (dict_size) o += r256(enc_dict_bytes(dict_size));
    L->offs = o;
    o += r256((size_t)L->nb_max * 8);
    L->sizes = o;
    o += r256((size_t)L->nb_max * 4);
    L->btiles = o;
    o += r256(((size_t)L->nb_max + ASM_TILE - 1) / ASM_TILE * 8);
    L->pool = o;
    o += (size_t)pool_units * 256 + L->wstride;
    L->total = o + 256; /* base alignment slack */
}

extern "C" size_t zxg_compress_batch_scratch_bytes(uint32_t max_frames, uint64_t max_total_src, uint32_t block_size,
                                                   int level, uint32_t dict_size) {
    if (zxg_init() != ZXC_OK || max_frames > CB_FRAMES_MAX || max_total_src > (1ull << 50)) return 0;
    /* the most any batch of max_frames frames of max_total_src bytes can take: input copies of r256(size + 64) bytes
     * and ceil(size / block_size) staging slots for each of at most m non-empty ones */
    const u64 m = max_frames < max_total_src ? max_frames : max_total_src;
    const u64 in = (max_total_src + 319ull * m) / 256;
    const u64 blocks = (max_total_src + m * (block_size - 1)) / block_size;
    const u64 need = in + blocks * (enc_staging_stride(block_size) / 256);
    if (need > CB_POOL_UNITS_MAX) return 0;
    /* and room for the encode slots of the warps that pool launches, beyond the one the layout always has */
    CBatchLayout L;
    cb_layout(max_frames, block_size, level, dict_size, need, &L);
    const u64 pool = need + (u64)(L.W - 1) * (L.wstride / 256);
    if (pool > CB_POOL_UNITS_MAX) return 0;
    cb_layout(max_frames, block_size, level, dict_size, pool, &L);
    return L.total;
}

extern "C" int zxg_compress_device_batch(const zxc_b200_frame_t* d_frames, uint32_t n_frames, uint32_t block_size,
                                         int level, int checksum, int seekable, const void* h_dict,
                                         uint32_t dict_size, const uint8_t* h_dict_huf_lens, const zxg_ddict_t* dd,
                                         const uint8_t* header, const uint8_t* eof, void* d_scratch,
                                         size_t scratch_size, int64_t* d_results, void* stream) {
    const int irc = zxg_init();
    if (irc != ZXC_OK) return irc;
    const u32 n = n_frames;
    if (n > CB_FRAMES_MAX) return ZXC_ERROR_MEMORY;
    const u32 dsz = h_dict && dict_size ? dict_size : 0;
    CBatchLayout L;
    cb_layout(n, block_size, level, dsz, 0, &L);
    if (L.total > scratch_size) return ZXC_ERROR_MEMORY;
    u64 lo = 0, hi = CB_POOL_UNITS_MAX; /* the largest pool whose layout fits */
    while (lo < hi) {
        const u64 mid = lo + (hi - lo + 1) / 2;
        cb_layout(n, block_size, level, dsz, mid, &L);
        if (L.total <= scratch_size) lo = mid;
        else hi = mid - 1;
    }
    cb_layout(n, block_size, level, dsz, lo, &L);
    cudaStream_t st = (cudaStream_t)stream;
    u8* base = (u8*)(((uintptr_t)d_scratch + 255) & ~(uintptr_t)255);
    CBatchArgs A;
    A.frames = d_frames;
    A.results = (long long*)d_results;
    A.st = (CBatchState*)base;
    A.F = (CBatchFrame*)(base + L.frames);
    A.first = (unsigned long long*)(base + L.first);
    A.ftiles = (unsigned long long*)(base + L.ftiles);
    A.btiles = (unsigned long long*)(base + L.btiles);
    A.offs = (unsigned long long*)(base + L.offs);
    A.sizes = (u32*)(base + L.sizes);
    A.staging = base + L.pool;
    A.pool_units = L.pool_units;
    A.wstride = L.wstride;
    A.n = n;
    A.nb_max = L.nb_max;
    A.warps = L.W;
    A.block_size = block_size;
    A.staging_stride = L.stride;
    A.checksum = checksum ? 1u : 0u;
    A.seekable = seekable ? 1u : 0u;
    memcpy(A.header, header, 16);
    memcpy(A.eof, eof, 8);
    EncodeParams P;
    memset(&P, 0, sizeof P);
    P.staging = A.staging;
    P.out_size = A.sizes;
    /* the W encode slots end at the room's end: slot g at scratch + g * wstride; those below the room never run */
    P.scratch = A.staging + (size_t)L.pool_units * 256 + L.wstride - (size_t)L.W * L.wstride;
    P.counter = &A.st->counter;
    if (dd || dsz) {
        const int rc = enc_stage_dict(P, base + L.dict, h_dict, dsz, level, h_dict_huf_lens, dd, true, st);
        if (rc != ZXC_OK) return rc;
    }
    P.scratch_stride = L.wstride;
    P.block_size = block_size;
    P.staging_stride = L.stride;
    P.level = (u32)level;
    P.checksum = A.checksum;
    P.dict_size = dd ? dd->dict_size : dsz;
    const u32 sms = (u32)(g_sm_count > 0 ? g_sm_count : 132);
    const u32 n_tiles = (n + ASM_TILE - 1) / ASM_TILE;
    const u32 per_frame = (n + CB_THREADS - 1) / CB_THREADS;
    const u32 b_tiles = (L.nb_max + ASM_TILE - 1) / ASM_TILE;
    const u32 by_warp = (L.nb_max + CB_THREADS / 32 - 1) / (CB_THREADS / 32);
    const u32 by_thread = (L.nb_max + CB_THREADS - 1) / CB_THREADS;
    zxc_cbatch_tiles<<<n_tiles, ASM_THREADS, 0, st>>>(A);
    zxc_cbatch_scan<<<1, ASM_SCAN_THREADS, 0, st>>>(A);
    zxc_cbatch_place<<<per_frame, CB_THREADS, 0, st>>>(A);
    zxc_cbatch_gather<<<by_warp < sms * 16 ? by_warp : sms * 16, CB_THREADS, 0, st>>>(A);
    const u32 grid = L.W >= ENC_WARPS_PER_CTA ? L.W / ENC_WARPS_PER_CTA : 1u;
    const u32 threads = L.W >= ENC_WARPS_PER_CTA ? ENC_CTA_THREADS : 32u * L.W;
    if (level >= 6) zxc_encode_batch_kernel<true><<<grid, threads, 0, st>>>(P, A);
    else zxc_encode_batch_kernel<false><<<grid, threads, 0, st>>>(P, A);
    zxc_cbatch_sums<<<b_tiles, ASM_THREADS, 0, st>>>(A);
    zxc_cbatch_bscan<<<1, ASM_SCAN_THREADS, 0, st>>>(A);
    zxc_cbatch_offsets<<<b_tiles, ASM_THREADS, 0, st>>>(A);
    zxc_cbatch_fit<<<per_frame, CB_THREADS, 0, st>>>(A);
    zxc_cbatch_blocks<<<by_thread < sms * 16 ? by_thread : sms * 16, CB_THREADS, 0, st>>>(A);
    __atomic_add_fetch(&g_launches, 10, __ATOMIC_RELAXED);
    launch_compact(A.staging, L.stride, A.offs, A.sizes, NULL /* absolute destinations */, L.nb_max, st);
    zxc_cbatch_finish<<<per_frame, CB_THREADS, 0, st>>>(A);
    __atomic_add_fetch(&g_launches, 1, __ATOMIC_RELAXED);
    return cudaGetLastError() == cudaSuccess ? ZXC_OK : ZXC_B200_ERROR_CUDA;
}

/* ------------------------------------------------------------------------- */
/* device-to-device decompress (zxc_b200_decompress_device): the frame walk, */
/* the decode and the verdict on the device (zxc_dplan.cuh)                  */
/* ------------------------------------------------------------------------- */
/* Scratch layout, from the caller's base rounded up to 256 bytes (every region 256-aligned):
 *   DPlanState | dictionary + its literal table | plan (J jobs) | decode jobs (J) | status (J x i32) |
 *   split sizes (J x i32) | SEK tile sums | split probe slots | decode scratch (per-warp regions, deferred list)
 * J = ceil(dst_capacity / ZXC_BLOCK_SIZE_MIN) + 2: every block but the last of a frame the reference's encoder
 * writes holds block_size >= ZXC_BLOCK_SIZE_MIN bytes, so such a frame fits the table when its output fits
 * dst_capacity. */
/* Builds a decode's dictionary region at d_region: the dictionary, then its literal table when h_huf is given, through
 * a pageable host copy, so the caller's dictionary has been read when the call returns, whatever memory it is in
 * (host_bounce). */
static int dec_build_dict(u8* d_region, const void* h_dict, u32 dict_size, const void* h_huf, cudaStream_t st) {
    const size_t dbytes = (size_t)dict_size + (h_huf ? ZXC_HUF_TABLE_SIZE : 0);
    u8* b = (u8*)host_bounce(h_dict, dict_size, dbytes);
    if (!b) return ZXC_ERROR_MEMORY;
    if (h_huf) memcpy(b + dict_size, h_huf, ZXC_HUF_TABLE_SIZE);
    const cudaError_t e = cudaMemcpyAsync(d_region, b, dbytes, cudaMemcpyHostToDevice, st);
    free(b);
    return e == cudaSuccess ? ZXC_OK : ZXC_B200_ERROR_CUDA;
}

/* A decode's dictionary and its literal table (when given): a prepared dictionary's decode region where it lies, or
 * the host dictionary built into the scratch's dictionary region at d_region.  Both device pointers stay NULL without
 * a dictionary. */
static int dec_stage_dict(u8* d_region, const zxg_dopts_t* o, cudaStream_t st, u8** d_dict, u8** d_huf) {
    *d_dict = (u8*)o->d_dict;
    *d_huf = (u8*)o->d_dict_huf;
    const u32 dict_size = o->dict_size;
    if (!o->dict || !dict_size) return ZXC_OK;
    *d_dict = d_region;
    if (o->dict_huf) *d_huf = d_region + dict_size;
    return dec_build_dict(d_region, o->dict, dict_size, o->dict_huf, st);
}

/* the device's share of the decode options, for a scratch sized for block size bs */
static DDecodeOpts dec_opts(const zxg_dopts_t* o, u32 bs) {
    DDecodeOpts d;
    d.max_block_size = bs;
    d.dict_id = o->dict_id;
    d.have_dict = (o->dict || o->d_dict) && o->dict_size ? 1u : 0u;
    d.huf_verdict = o->huf_verdict;
    d.checksum_enabled = o->checksum_enabled ? 1u : 0u;
    return d;
}

/* the largest v in [lo, hi] with fits(v), given fits(lo) and a fits that holds up to some value and not beyond: how
 * the calls below size their tables and windows to the scratch they are given */
template <class Fits>
static u64 largest_fit(u64 lo, u64 hi, Fits fits) {
    while (lo < hi) {
        const u64 mid = lo + (hi - lo + 1) / 2;
        if (fits(mid)) lo = mid;
        else hi = mid - 1;
    }
    return lo;
}

/* the largest block size b with fits(b) (0: none) */
template <class Fits>
static u32 largest_block_size(Fits fits) {
    for (u32 b = ZXC_BLOCK_SIZE_MAX; b >= ZXC_BLOCK_SIZE_MIN; b >>= 1)
        if (fits(b)) return b;
    return 0;
}

/* the general split's size probe (a rare path): one slot of bs + ZXF_TAIL_PAD per warp of the decode grid for
 * grid_jobs jobs, at most 256 MiB of them and at most J; returns the slots' bytes in the layout */
static size_t split_probe_slots(u32 bs, u32 grid_jobs, u64 J, u32* room, u32* probe_warps) {
    *room = bs + ZXF_TAIL_PAD;
    const u32 dec_warps = (u32)grid_for(grid_jobs) * WARPS_PER_CTA;
    const u32 by_room = (u32)(((size_t)256 << 20) / *room);
    u64 pw = dec_warps < by_room ? dec_warps : by_room;
    if (pw > J) pw = J;
    *probe_warps = pw ? (u32)pw : 1;
    return r256((size_t)*probe_warps * *room);
}

/* the general split's decode arguments: the plan's bases src and dst, its probe slots and the decode scratch */
static DSplitArgs split_args(const void* src, void* dst, u8* slots, u8* dec, const u8* d_dict, const u8* d_huf,
                             const zxg_dopts_t* o, u32 bs, u32 room, u32 probe_warps) {
    DSplitArgs D;
    D.src = (const u8*)src;
    D.dst = (u8*)dst;
    D.slots = slots;
    D.scratch = dec;
    D.dict = d_dict;
    D.dict_huf = d_huf;
    D.dict_size = d_dict ? o->dict_size : 0;
    D.scratch_stride = scratch_stride_for(bs);
    D.room = room;
    D.probe_warps = probe_warps;
    return D;
}

/* the general split's four launches for either kernel family (zxc_dplan.cuh, zxc_dbatch.cuh); they exit at once
 * unless a frame split */
template <class Ar>
static void launch_split(void (*decode)(Ar, DSplitArgs, u32), void (*scan)(Ar), void (*final)(Ar), const Ar& A,
                         const DSplitArgs& D, u32 dec_grid, u32 scan_grid, cudaStream_t st) {
    const u32 probe_grid = (D.probe_warps + WARPS_PER_CTA - 1) / WARPS_PER_CTA;
    decode<<<probe_grid, CTA_THREADS, DECODE_SMEM_BYTES, st>>>(A, D, 0);
    scan<<<scan_grid, ASM_SCAN_THREADS, 0, st>>>(A);
    decode<<<dec_grid, CTA_THREADS, DECODE_SMEM_BYTES, st>>>(A, D, 1);
    final<<<scan_grid, ASM_SCAN_THREADS, 0, st>>>(A);
    __atomic_add_fetch(&g_launches, 4, __ATOMIC_RELAXED);
}

/* one launch_decode per launch slot: block sizes up to bs, checksum verification off / on.  Slot s's jobs and status
 * words start at entry s * stride (stride 0: one table of n_jobs for every slot); only the slots with work have
 * counters preset below J on the device. */
static int launch_slot_decodes(const void* d_src, void* d_dst, const zxc_b200_job_t* jobs, i32* status, u32 n_jobs,
                               u64 stride, unsigned long long (*ctr)[4], const u8* d_dict, const u8* d_huf,
                               const zxg_dopts_t* o, u8* dec, size_t dec_bytes, u32 bs, cudaStream_t st) {
    for (u32 b = ZXC_BLOCK_SIZE_MIN; b <= bs; b <<= 1) {
        const u32 lg = (u32)__builtin_ctz(b) - ZXC_BLOCK_SIZE_MIN_LOG2;
        for (int v = 0; v <= (o->checksum_enabled ? 1 : 0); v++) {
            const u32 slot = lg * 2 + v;
            const int rc = launch_decode(d_src, d_dst, jobs + slot * stride, n_jobs, status + slot * stride, d_dict,
                                         o->dict_size, d_huf, dec, dec_bytes, b, v, ctr[slot], st, 1);
            if (rc != ZXC_OK) return rc;
        }
    }
    return ZXC_OK;
}

struct DevDecLayout {
    size_t dict, plan, jobs, status, sizes, tiles, slots, dec, dec_bytes, total;
    u32 J, probe_warps, room;
};
static bool dev_dec_layout(uint64_t dst_capacity, u32 block_size, DevDecLayout* L) {
    const uint64_t J64 = dst_capacity / ZXC_BLOCK_SIZE_MIN + (dst_capacity % ZXC_BLOCK_SIZE_MIN != 0) + 2;
    if (J64 > 0x7FFFFFFFull) return false;
    const u32 J = (u32)J64;
    size_t o = DP_STATE_BYTES;
    L->dict = o;
    o += r256((size_t)ZXC_DICT_SIZE_MAX + ZXC_HUF_TABLE_SIZE);
    L->plan = o;
    o += r256((size_t)J * sizeof(zxc_b200_job_t));
    L->jobs = o;
    o += r256((size_t)J * sizeof(zxc_b200_job_t));
    L->status = o;
    o += r256((size_t)J * 4);
    L->sizes = o;
    o += r256((size_t)J * 4);
    L->tiles = o;
    o += r256(((size_t)J + ASM_TILE - 1) / ASM_TILE * 8);
    L->slots = o;
    o += split_probe_slots(block_size, J, J, &L->room, &L->probe_warps);
    L->dec = o;
    L->dec_bytes = launch_scratch_bytes(J, block_size);
    o += L->dec_bytes;
    L->total = o + 256; /* base alignment slack */
    L->J = J;
    return true;
}

extern "C" size_t zxg_decompress_scratch_bytes(uint64_t dst_capacity, uint32_t block_size) {
    if (zxg_init() != ZXC_OK) return 0;
    DevDecLayout L;
    return dev_dec_layout(dst_capacity, block_size, &L) ? L.total : 0;
}

/* zxc_dplan.cuh's arguments over a DevDecLayout at base */
static DPlanArgs dplan_args(u8* base, const DevDecLayout& L, const void* d_src, uint64_t src_size,
                            uint64_t dst_capacity, u32 bs, const zxg_dopts_t* o, int64_t* d_result) {
    DPlanArgs A;
    A.src = (const u8*)d_src;
    A.src_size = src_size;
    A.dst_capacity = dst_capacity;
    A.plan = (zxc_b200_job_t*)(base + L.plan);
    A.jobs = (zxc_b200_job_t*)(base + L.jobs);
    A.status = (i32*)(base + L.status);
    A.sizes = (i32*)(base + L.sizes);
    A.tiles = (unsigned long long*)(base + L.tiles);
    A.st = (DPlanState*)base;
    A.result = (long long*)d_result;
    A.J = L.J;
    A.o = dec_opts(o, bs);
    return A;
}

/* the frame's plan: probe, SEK-guided plan, walk, and the job table */
static void launch_dplan(const DPlanArgs& A, cudaStream_t st) {
    const u32 n_tiles = (A.J + ASM_TILE - 1) / ASM_TILE;
    const u32 per_job = (A.J + DP_THREADS - 1) / DP_THREADS;
    zxc_dplan_probe<<<1, 1, 0, st>>>(A);
    zxc_dplan_sek_tiles<<<n_tiles, ASM_THREADS, 0, st>>>(A);
    zxc_dplan_sek_scan<<<1, ASM_SCAN_THREADS, 0, st>>>(A);
    zxc_dplan_sek_blocks<<<n_tiles, ASM_THREADS, 0, st>>>(A);
    zxc_dplan_walk<<<1, 32, 0, st>>>(A);
    zxc_dplan_place<<<per_job, DP_THREADS, 0, st>>>(A);
    __atomic_add_fetch(&g_launches, 6, __ATOMIC_RELAXED);
}

/* the first failing job, then zxc_decompress's verdict or the general split's go-ahead */
static void launch_dplan_verdict(const DPlanArgs& A, cudaStream_t st) {
    zxc_dplan_check<<<(A.J + DP_THREADS - 1) / DP_THREADS, DP_THREADS, 0, st>>>(A);
    zxc_dplan_decide<<<1, 1, 0, st>>>(A);
    __atomic_add_fetch(&g_launches, 2, __ATOMIC_RELAXED);
}

/* the single frame's general split, its plan's offsets over src and dst */
static void launch_dsplit(const DPlanArgs& A, const DevDecLayout& L, u8* base, const void* src, void* dst,
                          const u8* d_dict, const u8* d_huf, const zxg_dopts_t* o, u32 bs, cudaStream_t st) {
    const DSplitArgs D = split_args(src, dst, base + L.slots, base + L.dec, d_dict, d_huf, o, bs, L.room,
                                    L.probe_warps);
    launch_split(d_dict ? zxc_dsplit_decode<true> : zxc_dsplit_decode<false>, zxc_dsplit_scan, zxc_dsplit_final, A,
                 D, (u32)grid_for(L.J), 1, st);
}

extern "C" int zxg_decompress_device(const void* d_src, uint64_t src_size, void* d_dst, uint64_t dst_capacity,
                                     const zxg_dopts_t* o, void* d_scratch, size_t scratch_size, int64_t* d_result,
                                     void* stream) {
    const int irc = zxg_init();
    if (irc != ZXC_OK) return irc;
    /* the largest block size this scratch was sized for */
    DevDecLayout L;
    const u32 bs = largest_block_size([&](u32 b) {
        return dev_dec_layout(dst_capacity, b, &L) && L.total <= scratch_size;
    });
    if (!bs) return ZXC_ERROR_MEMORY;
    cudaStream_t st = (cudaStream_t)stream;
    u8* base = (u8*)(((uintptr_t)d_scratch + 255) & ~(uintptr_t)255);
    u8 *d_dict, *d_huf;
    const int drc = dec_stage_dict(base + L.dict, o, st, &d_dict, &d_huf);
    if (drc != ZXC_OK) return drc;
    const DPlanArgs A = dplan_args(base, L, d_src, src_size, dst_capacity, bs, o, d_result);
    launch_dplan(A, st);
    const int rc = launch_slot_decodes(d_src, d_dst, A.jobs, A.status, L.J, 0, A.st->ctr, d_dict, d_huf, o,
                                       base + L.dec, L.dec_bytes, bs, st);
    if (rc != ZXC_OK) return rc;
    launch_dplan_verdict(A, st);
    launch_dsplit(A, L, base, d_src, d_dst, d_dict, d_huf, o, bs, st);
    return cudaGetLastError() == cudaSuccess ? ZXC_OK : ZXC_B200_ERROR_CUDA;
}

/* ------------------------------------------------------------------------- */
/* in-place decode of a device-resident frame (zxc_b200_decompress_inplace_  */
/* device: kernels in zxc_dinplace.cuh)                                      */
/* ------------------------------------------------------------------------- */
/* Scratch layout: zxc_b200_decompress_device's (DevDecLayout for buffer_capacity and B), then, every region
 * 256-aligned: the hazard flag | round starts (R_max + 1 x u64) | two round tables (Jr jobs) | their status arrays
 * (Jr x i32) | the staging area of W + O + 64 bytes.  O = B + 12 (a RAW block with its checksum: the largest block the
 * reference's encoder writes at block size B), Jr = min(J, W / 8 + 1), R_max = ceil(buffer_capacity / W_min) + 1 with
 * W_min the smallest window. */
struct InplaceLayout {
    DevDecLayout d;
    size_t hazard, rstart, rjobs[2], rstatus[2], staging, total;
    u64 W, O;
    u32 bs, Jr;
};
/* windows are whole multiples of IP_WINDOW_UNIT, from W_min = 2 (B + O) rounded up to the unit, to the buffer's
 * capacity rounded up to it; a scratch sized for a window then gives exactly that window (unless a larger B fits) */
#define IP_WINDOW_UNIT 4096ull
static u64 ip_round_up(u64 v) { return (v + IP_WINDOW_UNIT - 1) / IP_WINDOW_UNIT * IP_WINDOW_UNIT; }
static u64 ip_window_min(u32 bs) { return ip_round_up(2ull * (bs + (u64)bs + ZXF_BLOCK_HDR + ZXF_BLOCK_CKS)); }
static u64 ip_window_max(uint64_t cap, u32 bs) {
    const u64 w = ip_round_up(cap);
    return w > ip_window_min(bs) ? w : ip_window_min(bs);
}

static bool ip_layout(uint64_t cap, u32 bs, u64 W, InplaceLayout* L) {
    if (!dev_dec_layout(cap, bs, &L->d)) return false;
    const u64 w_min = ip_window_min(bs);
    W = W < w_min ? w_min : (W > ip_window_max(cap, bs) ? ip_window_max(cap, bs) : ip_round_up(W));
    const u64 r_max = (cap + w_min - 1) / w_min + 1;
    const u64 jr = W / ZXF_BLOCK_HDR + 1 < L->d.J ? W / ZXF_BLOCK_HDR + 1 : L->d.J;
    size_t o = L->d.total - 256; /* DevDecLayout's end, before its base alignment slack */
    L->hazard = o;
    o += 256;
    L->rstart = o;
    o += r256((size_t)(r_max + 1) * 8);
    for (int t = 0; t < 2; t++) {
        L->rjobs[t] = o;
        o += r256((size_t)jr * sizeof(zxc_b200_job_t));
        L->rstatus[t] = o;
        o += r256((size_t)jr * 4);
    }
    L->O = (u64)bs + ZXF_BLOCK_HDR + ZXF_BLOCK_CKS;
    L->staging = o;
    o += r256((size_t)(W + L->O + 64));
    L->total = o + 256;
    L->W = W;
    L->bs = bs;
    L->Jr = (u32)jr;
    return true;
}

extern "C" size_t zxg_decompress_inplace_scratch_bytes(uint64_t buffer_capacity, uint32_t block_size, uint64_t window) {
    if (zxg_init() != ZXC_OK) return 0;
    InplaceLayout L;
    return ip_layout(buffer_capacity, block_size, window, &L) ? L.total : 0;
}

/* B and W from the scratch size: the largest B whose layout with the smallest window fits, then the largest window
 * (up to the whole buffer) that fits at B, both in window units */
static bool ip_choose(uint64_t cap, size_t scratch_size, InplaceLayout* L) {
    const auto fits = [&](u32 b, u64 W) { return ip_layout(cap, b, W, L) && L->total <= scratch_size; };
    const u32 bs = largest_block_size([&](u32 b) { return fits(b, 0); });
    if (!bs) return false;
    const u64 units = largest_fit(L->W / IP_WINDOW_UNIT, ip_window_max(cap, bs) / IP_WINDOW_UNIT,
                                  [&](u64 u) { return fits(bs, u * IP_WINDOW_UNIT); });
    return ip_layout(cap, bs, units * IP_WINDOW_UNIT, L);
}

extern "C" int zxg_decompress_inplace_device(void* d_buffer, uint64_t buffer_capacity, uint64_t comp_size,
                                             const zxg_dopts_t* o, void* d_scratch, size_t scratch_size,
                                             int64_t* d_result, void* stream) {
    const int irc = zxg_init();
    if (irc != ZXC_OK) return irc;
    InplaceLayout L;
    if (!ip_choose(buffer_capacity, scratch_size, &L)) return ZXC_ERROR_MEMORY;
    const u32 bs = L.bs;
    const u64 W = L.W;
    const u32 R = (u32)((comp_size + W - 1) / W);
    cudaStream_t st = (cudaStream_t)stream;
    u8* base = (u8*)(((uintptr_t)d_scratch + 255) & ~(uintptr_t)255);
    u8 *d_dict, *d_huf;
    const int drc = dec_stage_dict(base + L.d.dict, o, st, &d_dict, &d_huf);
    if (drc != ZXC_OK) return drc;
    u8* buf = (u8*)d_buffer;
    const u64 off = buffer_capacity - comp_size; /* the frame lies flush-right */
    DInplaceArgs I;
    I.a = dplan_args(base, L.d, buf + off, comp_size, buffer_capacity, bs, o, d_result);
    I.hazard = (unsigned int*)(base + L.hazard);
    I.rstart = (unsigned long long*)(base + L.rstart);
    for (int t = 0; t < 2; t++) {
        I.rjobs[t] = (zxc_b200_job_t*)(base + L.rjobs[t]);
        I.rstatus[t] = (i32*)(base + L.rstatus[t]);
    }
    I.base = off;
    I.W = W;
    I.O = L.O;
    I.R = R;
    I.Jr = L.Jr;
    launch_dplan(I.a, st);
    zxc_dinplace_probe<<<1, 1, 0, st>>>(I);
    const u64 plan_threads = (u64)L.d.J > (u64)R + 1 ? L.d.J : (u64)R + 1;
    zxc_dinplace_plan<<<(u32)((plan_threads + DI_THREADS - 1) / DI_THREADS), DI_THREADS, 0, st>>>(I);
    __atomic_add_fetch(&g_launches, 2, __ATOMIC_RELAXED);
    /* round k: frame bytes [k W - 8, min(k W + W + O + 8, comp_size)) into the staging area, frame byte x at
     * staging + 8 + x - k W, then the round's jobs and their decode from there */
    u8* staging = base + L.staging;
    const u32 round_grid = (L.Jr + DI_THREADS - 1) / DI_THREADS;
    for (u32 k = 0; k < R; k++) {
        const u64 w = (u64)k * W;
        const u64 lo = w >= 8 ? w - 8 : 0;
        const u64 hi = w + W + L.O + 8 < comp_size ? w + W + L.O + 8 : comp_size;
        if (cudaMemcpyAsync(staging + 8 + lo - w, buf + off + lo, (size_t)(hi - lo), cudaMemcpyDeviceToDevice, st) !=
            cudaSuccess)
            return ZXC_B200_ERROR_CUDA;
        zxc_dinplace_round<<<round_grid, DI_THREADS, 0, st>>>(I, k);
        __atomic_add_fetch(&g_launches, 1, __ATOMIC_RELAXED);
        const int rc = launch_slot_decodes(staging + 8 - w, buf, I.rjobs[k & 1], I.rstatus[k & 1], L.Jr, 0,
                                           I.a.st->ctr, d_dict, d_huf, o, base + L.d.dec, L.d.dec_bytes, bs, st);
        if (rc != ZXC_OK) return rc;
    }
    zxc_dinplace_round<<<round_grid, DI_THREADS, 0, st>>>(I, R);
    __atomic_add_fetch(&g_launches, 1, __ATOMIC_RELAXED);
    launch_dplan_verdict(I.a, st);
    zxc_dinplace_nosplit<<<1, 1, 0, st>>>(I);
    __atomic_add_fetch(&g_launches, 1, __ATOMIC_RELAXED);
    /* the split runs with one round only: the whole frame is then in the staging area */
    launch_dsplit(I.a, L.d, base, staging + 8, buf, d_dict, d_huf, o, bs, st);
    return cudaGetLastError() == cudaSuccess ? ZXC_OK : ZXC_B200_ERROR_CUDA;
}

/* ------------------------------------------------------------------------- */
/* many device-resident frames in one call (zxc_b200_decompress_device_batch: */
/* kernels in zxc_dbatch.cuh)                                                */
/* ------------------------------------------------------------------------- */
/* Scratch layout, from the caller's base rounded up to 256 bytes (every region 256-aligned):
 *   DBatchState | dictionary + its literal table | frames (n x DBatchFrame) | table offsets (n x u64) | tile sums |
 *   slot tile sums (n_slots per tile) | plan (Jt jobs) | split sizes (Jt x i32) | slot windows (n_slots x Jt jobs) |
 *   slot status (n_slots x Jt x i32) | split probe slots | decode scratch (per-warp regions, deferred list)
 * n_slots = 2 per block size from 4 KiB up to B (checksum verification off / on).  The per-warp regions are sized for
 * the full resident grid at B, whatever Jt: so B, which the call finds as the largest block size whose layout with
 * the smallest table fits the scratch, is the block size the scratch was sized for unless the table's share is larger
 * than the step in the per-warp regions to the next block size. */
struct DBatchLayout {
    size_t dict, frames, base, tiles, stiles, plan, sizes, jobs, status, slots, dec, dec_bytes, total;
    u32 n_slots, probe_warps, room;
    u64 Jt;
};
#define DB_J_MAX 0x7FFFFFFFull
#define DB_FRAMES_MAX (1u << 30)

static void db_layout(u32 n, u64 Jt, u32 bs, DBatchLayout* L) {
    const size_t n_tiles = ((size_t)n + ASM_TILE - 1) / ASM_TILE;
    L->n_slots = ((u32)__builtin_ctz(bs) - ZXC_BLOCK_SIZE_MIN_LOG2 + 1) * 2;
    size_t o = DB_STATE_BYTES;
    L->dict = o;
    o += r256((size_t)ZXC_DICT_SIZE_MAX + ZXC_HUF_TABLE_SIZE);
    L->frames = o;
    o += r256((size_t)n * sizeof(DBatchFrame));
    L->base = o;
    o += r256((size_t)n * 8);
    L->tiles = o;
    o += r256(n_tiles * 8);
    L->stiles = o;
    o += r256(n_tiles * L->n_slots * 8);
    L->plan = o;
    o += r256((size_t)Jt * sizeof(zxc_b200_job_t));
    L->sizes = o;
    o += r256((size_t)Jt * 4);
    L->jobs = o;
    o += r256((size_t)L->n_slots * Jt * sizeof(zxc_b200_job_t));
    L->status = o;
    o += r256((size_t)L->n_slots * Jt * 4);
    L->slots = o;
    o += split_probe_slots(bs, (u32)DB_J_MAX, Jt, &L->room, &L->probe_warps);
    L->dec = o;
    L->dec_bytes = launch_scratch_bytes((u32)DB_J_MAX, bs);
    L->total = o + L->dec_bytes + 256; /* base alignment slack */
    L->Jt = Jt;
}

extern "C" size_t zxg_decompress_batch_scratch_bytes(uint32_t max_frames, uint64_t max_total_capacity,
                                                     uint32_t block_size) {
    if (zxg_init() != ZXC_OK || max_frames > DB_FRAMES_MAX) return 0;
    const u64 Jt = max_total_capacity / ZXC_BLOCK_SIZE_MIN + (max_total_capacity % ZXC_BLOCK_SIZE_MIN != 0) +
                   3ull * max_frames;
    if (Jt > DB_J_MAX) return 0;
    DBatchLayout L;
    db_layout(max_frames, Jt ? Jt : 1, block_size, &L);
    return L.total;
}

extern "C" int zxg_decompress_device_batch(const zxc_b200_frame_t* d_frames, uint32_t n_frames, const zxg_dopts_t* o,
                                           void* d_scratch, size_t scratch_size, int64_t* d_results, void* stream) {
    const int irc = zxg_init();
    if (irc != ZXC_OK) return irc;
    const u32 n = n_frames;
    if (n > DB_FRAMES_MAX) return ZXC_ERROR_MEMORY;
    const u64 J_min = 3ull * n;
    /* the largest block size whose layout with the smallest table fits, then the largest table at it */
    DBatchLayout L;
    const auto fits = [&](u32 b, u64 Jt) {
        db_layout(n, Jt, b, &L);
        return L.total <= scratch_size;
    };
    const u32 bs = largest_block_size([&](u32 b) { return fits(b, J_min); });
    if (!bs) return ZXC_ERROR_MEMORY;
    db_layout(n, largest_fit(J_min, DB_J_MAX, [&](u64 Jt) { return fits(bs, Jt); }), bs, &L);
    cudaStream_t st = (cudaStream_t)stream;
    u8* base = (u8*)(((uintptr_t)d_scratch + 255) & ~(uintptr_t)255);
    u8 *d_dict, *d_huf;
    const int drc = dec_stage_dict(base + L.dict, o, st, &d_dict, &d_huf);
    if (drc != ZXC_OK) return drc;
    DBatchState* S = (DBatchState*)base;
    DBatchArgs A;
    A.frames = d_frames;
    A.results = (long long*)d_results;
    A.st = S;
    A.F = (DBatchFrame*)(base + L.frames);
    A.base = (unsigned long long*)(base + L.base);
    A.tiles = (unsigned long long*)(base + L.tiles);
    A.stiles = (unsigned long long*)(base + L.stiles);
    A.plan = (zxc_b200_job_t*)(base + L.plan);
    A.sizes = (i32*)(base + L.sizes);
    A.jobs = (zxc_b200_job_t*)(base + L.jobs);
    A.status = (i32*)(base + L.status);
    A.Jt = L.Jt;
    A.n = n;
    A.n_slots = L.n_slots;
    A.o = dec_opts(o, bs);
    const u32 n_tiles = (n + ASM_TILE - 1) / ASM_TILE;
    const u32 per_frame = (n + DB_THREADS - 1) / DB_THREADS;
    const u32 per_cta = n < 4096 ? n : 4096; /* grid-stride over frames, one CTA each */
    const u64 by_entry = (L.Jt + DB_THREADS - 1) / DB_THREADS;
    const u32 per_entry = (u32)(by_entry < 16384 ? by_entry : 16384);
    zxc_dbatch_tiles<<<n_tiles, ASM_THREADS, 0, st>>>(A);
    zxc_dbatch_scan<<<1, ASM_SCAN_THREADS, 0, st>>>(A);
    zxc_dbatch_probe<<<per_frame, DB_THREADS, 0, st>>>(A);
    zxc_dbatch_sek<<<per_cta, ASM_THREADS, 0, st>>>(A);
    zxc_dbatch_walk<<<(u32)(((u64)n * 32 + DB_THREADS - 1) / DB_THREADS), DB_THREADS, 0, st>>>(A);
    zxc_dbatch_count<<<n_tiles, ASM_THREADS, 0, st>>>(A);
    zxc_dbatch_slots<<<1, ASM_SCAN_THREADS, 0, st>>>(A);
    zxc_dbatch_place<<<per_entry, DB_THREADS, 0, st>>>(A);
    __atomic_add_fetch(&g_launches, 8, __ATOMIC_RELAXED);
    if (cudaGetLastError() != cudaSuccess) return ZXC_B200_ERROR_CUDA;
    /* each launch slot over its own window */
    u8* dec = base + L.dec;
    const int rc = launch_slot_decodes(NULL, NULL, A.jobs, A.status, (u32)L.Jt, L.Jt, S->ctr, d_dict, d_huf, o, dec,
                                       L.dec_bytes, bs, st);
    if (rc != ZXC_OK) return rc;
    zxc_dbatch_check<<<per_entry, DB_THREADS, 0, st>>>(A);
    zxc_dbatch_decide<<<per_frame, DB_THREADS, 0, st>>>(A);
    __atomic_add_fetch(&g_launches, 2, __ATOMIC_RELAXED);
    /* the jobs' offsets are device addresses: the split's bases are zero */
    const DSplitArgs D = split_args(NULL, NULL, base + L.slots, dec, d_dict, d_huf, o, bs, L.room, L.probe_warps);
    launch_split(d_dict ? zxc_dbatch_split<true> : zxc_dbatch_split<false>, zxc_dbatch_split_scan,
                 zxc_dbatch_split_final, A, D, (u32)grid_for((u32)L.Jt), n < 1024 ? n : 1024, st);
    return cudaGetLastError() == cudaSuccess ? ZXC_OK : ZXC_B200_ERROR_CUDA;
}

/* ------------------------------------------------------------------------- */
/* the block API in HBM (zxc_b200_compress_blocks_device,                    */
/* zxc_b200_decompress_blocks_device: kernels in zxc_blocks.cuh)             */
/* ------------------------------------------------------------------------- */
/* Compress scratch layout, from the caller's base rounded up to 256 bytes (every region 256-aligned):
 *   BlocksCState | items (n x BlocksCItem) | tile sums (2 per tile) | dictionary region (with a dictionary) | room
 * The room holds the pool from its start and the encode slots from its end (zxc_blocks.cuh). */
static size_t bk_clayout(u32 n, u32 dict_size, size_t* items, size_t* tiles, size_t* dict) {
    const size_t n_tiles = ((size_t)n + ASM_TILE - 1) / ASM_TILE;
    size_t o = BK_STATE_BYTES;
    *items = o;
    o += r256((size_t)n * sizeof(BlocksCItem));
    *tiles = o;
    o += r256(n_tiles * 16);
    *dict = o;
    if (dict_size) o += r256(enc_dict_bytes(dict_size));
    return o; /* the room's offset */
}

/* encode warps of a call over n items: one per item up to the resident grid, whole CTAs from ENC_WARPS_PER_CTA up */
static u32 bk_warps(u32 n) {
    const u32 resident = (u32)(g_sm_count > 0 ? g_sm_count : 132) * ENC_CTAS_PER_SM * ENC_WARPS_PER_CTA;
    u32 W = n < resident ? n : resident;
    if (W >= ENC_WARPS_PER_CTA) W -= W % ENC_WARPS_PER_CTA;
    return W ? W : 1u;
}

extern "C" size_t zxg_compress_blocks_scratch_bytes(uint32_t max_blocks, uint64_t max_total_src, uint32_t max_src_size,
                                                    int level, uint32_t dict_size) {
    if (zxg_init() != ZXC_OK || max_blocks > CB_FRAMES_MAX || max_total_src > (1ull << 50) ||
        max_src_size > ZXC_BLOCK_SIZE_MAX)
        return 0;
    size_t items, tiles, dict;
    const size_t room = bk_clayout(max_blocks, dict_size, &items, &tiles, &dict);
    /* an n-byte item's share is r256(n + 64) + r256(n + 12) <= 2 n + 586 bytes, for at most k non-empty items */
    const u64 k = max_blocks < max_total_src ? max_blocks : max_total_src;
    const u64 pool = r256(2 * max_total_src + 586 * k);
    /* no more encode slots than items that can be non-empty: a scratch for no bytes holds one, the call's minimum */
    const size_t ws = enc_layout((u32)zxf_block_size_ceil(max_src_size), level).total;
    const u32 W = bk_warps(k < max_blocks ? (u32)k : max_blocks);
    return room + pool + (size_t)W * ws + 256; /* base alignment slack */
}

extern "C" int zxg_compress_blocks_device(const zxc_b200_frame_t* d_items, uint32_t n_items, int level, int checksum,
                                          const void* h_dict, uint32_t dict_size, const zxg_ddict_t* dd,
                                          void* d_scratch, size_t scratch_size, int64_t* d_results, void* stream) {
    const int irc = zxg_init();
    if (irc != ZXC_OK) return irc;
    const u32 n = n_items;
    if (n > CB_FRAMES_MAX) return ZXC_ERROR_MEMORY;
    const u32 dsz = h_dict && dict_size ? dict_size : 0;
    size_t items, tiles, dict;
    const size_t room = bk_clayout(n, dsz, &items, &tiles, &dict);
    if (scratch_size < room + enc_layout(ZXC_BLOCK_SIZE_MIN, level).total + 256) return ZXC_ERROR_MEMORY;
    cudaStream_t st = (cudaStream_t)stream;
    u8* base = (u8*)(((uintptr_t)d_scratch + 255) & ~(uintptr_t)255);
    BlocksCArgs A;
    A.items = d_items;
    A.results = (long long*)d_results;
    A.st = (BlocksCState*)base;
    A.I = (BlocksCItem*)(base + items);
    A.tiles = (unsigned long long*)(base + tiles);
    A.room = base + room;
    A.room_bytes = (scratch_size - 256 - room) & ~(size_t)255;
    for (u32 c = 0; c < BK_CLASSES; c++) A.wstride[c] = enc_layout(ZXC_BLOCK_SIZE_MIN << c, level).total;
    A.n = n;
    A.warps = bk_warps(n);
    EncodeParams P;
    memset(&P, 0, sizeof P);
    P.counter = &A.st->counter;
    if (dd || dsz) { /* the block API attaches no shared literal table */
        const int rc = enc_stage_dict(P, base + dict, h_dict, dsz, level, NULL, dd, false, st);
        if (rc != ZXC_OK) return rc;
    }
    P.level = (u32)level;
    P.checksum = checksum ? 1u : 0u;
    P.dict_size = dd ? dd->dict_size : dsz;
    const u32 sms = (u32)(g_sm_count > 0 ? g_sm_count : 132);
    const u32 n_tiles = (n + ASM_TILE - 1) / ASM_TILE;
    const u32 by_warp = (n + BK_THREADS / 32 - 1) / (BK_THREADS / 32);
    const u32 wgrid = by_warp < sms * 16 ? by_warp : sms * 16;
    zxc_blocks_ctiles<<<n_tiles, ASM_THREADS, 0, st>>>(A);
    zxc_blocks_cscan<<<1, 1, 0, st>>>(A);
    zxc_blocks_cgather<<<wgrid, BK_THREADS, 0, st>>>(A);
    const u32 grid = A.warps >= ENC_WARPS_PER_CTA ? A.warps / ENC_WARPS_PER_CTA : 1u;
    const u32 threads = A.warps >= ENC_WARPS_PER_CTA ? ENC_CTA_THREADS : 32u * A.warps;
    if (level >= 6) zxc_blocks_encode<true><<<grid, threads, 0, st>>>(P, A);
    else zxc_blocks_encode<false><<<grid, threads, 0, st>>>(P, A);
    zxc_blocks_cfinish<<<wgrid, BK_THREADS, 0, st>>>(A);
    __atomic_add_fetch(&g_launches, 5, __ATOMIC_RELAXED);
    return cudaGetLastError() == cudaSuccess ? ZXC_OK : ZXC_B200_ERROR_CUDA;
}

/* Decompress scratch layout, from the caller's base rounded up to 256 bytes (every region 256-aligned):
 *   DBatchState | dictionary region | items (n x BlocksDItem) | slot tile sums (n_slots per tile) | slot windows
 *   (n_slots x n jobs) | slot status (n_slots x n x i32) | decode scratch for n jobs at B
 * n_slots = 2 per block size from 4 KiB up to B (checksum verification off / on, dp_slot's numbering). */
struct BlocksDLayout {
    size_t dict, items, stiles, jobs, status, dec, dec_bytes, total;
    u32 n_slots;
};
static void bk_dlayout(u32 n, u32 bs, BlocksDLayout* L) {
    const size_t n_tiles = ((size_t)n + ASM_TILE - 1) / ASM_TILE;
    L->n_slots = ((u32)__builtin_ctz(bs) - ZXC_BLOCK_SIZE_MIN_LOG2 + 1) * 2;
    size_t o = DB_STATE_BYTES;
    L->dict = o;
    o += r256((size_t)ZXC_DICT_SIZE_MAX);
    L->items = o;
    o += r256((size_t)n * sizeof(BlocksDItem));
    L->stiles = o;
    o += r256(n_tiles * L->n_slots * 8);
    L->jobs = o;
    o += r256((size_t)L->n_slots * n * sizeof(zxc_b200_job_t));
    L->status = o;
    o += r256((size_t)L->n_slots * n * 4);
    L->dec = o;
    L->dec_bytes = launch_scratch_bytes(n ? n : 1, bs);
    L->total = o + L->dec_bytes + 256; /* base alignment slack */
}

extern "C" size_t zxg_decompress_blocks_scratch_bytes(uint32_t max_blocks, uint64_t max_dst_capacity) {
    if (zxg_init() != ZXC_OK || max_blocks > DB_FRAMES_MAX) return 0;
    BlocksDLayout L;
    bk_dlayout(max_blocks, (u32)zxf_block_size_ceil(max_dst_capacity), &L);
    return L.total;
}

extern "C" int zxg_decompress_blocks_device(const zxc_b200_frame_t* d_items, uint32_t n_items, const zxg_dopts_t* o,
                                            int safe, void* d_scratch, size_t scratch_size, int64_t* d_results,
                                            void* stream) {
    const int irc = zxg_init();
    if (irc != ZXC_OK) return irc;
    const u32 n = n_items;
    if (n > DB_FRAMES_MAX) return ZXC_ERROR_MEMORY;
    BlocksDLayout L;
    const u32 bs = largest_block_size([&](u32 b) {
        bk_dlayout(n, b, &L);
        return L.total <= scratch_size;
    });
    if (!bs) return ZXC_ERROR_MEMORY;
    bk_dlayout(n, bs, &L);
    cudaStream_t st = (cudaStream_t)stream;
    u8* base = (u8*)(((uintptr_t)d_scratch + 255) & ~(uintptr_t)255);
    u8 *d_dict, *d_huf;
    const int drc = dec_stage_dict(base + L.dict, o, st, &d_dict, &d_huf);
    if (drc != ZXC_OK) return drc;
    DBatchState* S = (DBatchState*)base;
    BlocksDArgs A;
    A.items = d_items;
    A.results = (long long*)d_results;
    A.st = S;
    A.I = (BlocksDItem*)(base + L.items);
    A.stiles = (unsigned long long*)(base + L.stiles);
    A.jobs = (zxc_b200_job_t*)(base + L.jobs);
    A.status = (i32*)(base + L.status);
    A.cap_max = safe ? (u64)ZXC_BLOCK_SIZE_MAX : (u64)ZXC_BLOCK_SIZE_MAX + ZXF_TAIL_PAD;
    A.n = n;
    A.n_slots = L.n_slots;
    A.bs = bs;
    A.verify = o->checksum_enabled ? 1u : 0u;
    /* zxc_dbatch_slots reads the state, the slot tile sums and the window size n */
    DBatchArgs D;
    memset(&D, 0, sizeof D);
    D.st = S;
    D.stiles = A.stiles;
    D.Jt = n;
    D.n = n;
    D.n_slots = L.n_slots;
    const u32 per_item = (n + BK_THREADS - 1) / BK_THREADS;
    zxc_blocks_dcount<<<(n + ASM_TILE - 1) / ASM_TILE, ASM_THREADS, 0, st>>>(A);
    zxc_dbatch_slots<<<1, ASM_SCAN_THREADS, 0, st>>>(D);
    zxc_blocks_dplace<<<per_item, BK_THREADS, 0, st>>>(A);
    __atomic_add_fetch(&g_launches, 3, __ATOMIC_RELAXED);
    if (cudaGetLastError() != cudaSuccess) return ZXC_B200_ERROR_CUDA;
    /* the jobs' offsets are device addresses: the decode's bases are zero */
    const int rc = launch_slot_decodes(NULL, NULL, A.jobs, A.status, n, n, S->ctr, d_dict, NULL, o, base + L.dec,
                                       L.dec_bytes, bs, st);
    if (rc != ZXC_OK) return rc;
    zxc_blocks_dfinish<<<per_item, BK_THREADS, 0, st>>>(A);
    __atomic_add_fetch(&g_launches, 1, __ATOMIC_RELAXED);
    return cudaGetLastError() == cudaSuccess ? ZXC_OK : ZXC_B200_ERROR_CUDA;
}

/* ------------------------------------------------------------------------- */
/* push streams in HBM (zxc_b200_cstream_device / _dstream_device:           */
/* zxc_pstream.c drives these, kernels in zxc_pstream_device.cuh)            */
/* ------------------------------------------------------------------------- */
static int ps_cuda(cudaError_t e) {
    if (e == cudaSuccess) return ZXC_OK;
    fprintf(stderr, "libzxc (CUDA build): device stream step failed: %s\n", cudaGetErrorString(e));
    cudaGetLastError();
    return ZXC_B200_ERROR_CUDA;
}

extern "C" int zxg_d2d_async(void* d_dst, const void* d_src, size_t bytes, void* stream) {
    if (bytes == 0) return ZXC_OK;
    return ps_cuda(cudaMemcpyAsync(d_dst, d_src, bytes, cudaMemcpyDeviceToDevice, (cudaStream_t)stream));
}

extern "C" int zxg_h2d_async(void* d_dst, const void* h_src, size_t bytes, void* stream) {
    if (bytes == 0) return ZXC_OK;
    return ps_cuda(cudaMemcpyAsync(d_dst, h_src, bytes, cudaMemcpyHostToDevice, (cudaStream_t)stream));
}

extern "C" int zxg_memset_async(void* d_dst, int v, size_t bytes, void* stream) {
    if (bytes == 0) return ZXC_OK;
    return ps_cuda(cudaMemsetAsync(d_dst, v, bytes, (cudaStream_t)stream));
}

extern "C" void* zxg_host_alloc(size_t bytes) {
    void* h = NULL;
    if (cudaMallocHost(&h, bytes) != cudaSuccess) {
        cudaGetLastError();
        return NULL;
    }
    return h;
}

extern "C" void zxg_host_free(void* h) {
    if (h) cudaFreeHost(h);
}

extern "C" int zxg_stream_sync(void* stream) { return ps_cuda(cudaStreamSynchronize((cudaStream_t)stream)); }

extern "C" int zxg_ps_walk(const void* d_src, uint64_t size, uint32_t max_blocks, uint64_t bound, int has_checksum,
                           zxg_psblk_t* d_out, zxg_psblk_t* h_out, uint32_t* n_out, void* stream) {
    cudaStream_t st = (cudaStream_t)stream;
    u32* d_n = (u32*)(d_out + max_blocks + 1);
    zxc_ps_walk<<<1, 32, 0, st>>>((const u8*)d_src, size, max_blocks, bound, has_checksum ? 1u : 0u, d_out, d_n);
    __atomic_add_fetch(&g_launches, 1, __ATOMIC_RELAXED);
    /* the entries and the count are one region: one copy, one synchronisation */
    const size_t bytes = ((size_t)max_blocks + 1) * sizeof(zxg_psblk_t) + sizeof(u32);
    int rc = ps_cuda(cudaGetLastError());
    if (rc == ZXC_OK) rc = ps_cuda(cudaMemcpyAsync(h_out, d_out, bytes, cudaMemcpyDeviceToHost, st));
    if (rc == ZXC_OK) rc = ps_cuda(cudaStreamSynchronize(st));
    if (rc == ZXC_OK) memcpy(n_out, (const u8*)h_out + bytes - sizeof(u32), sizeof(u32));
    return rc;
}

extern "C" size_t zxg_ps_decode_scratch_bytes(uint32_t n_jobs, uint32_t block_size) {
    return launch_scratch_bytes(n_jobs, block_size);
}

extern "C" size_t zxg_ps_encode_scratch_bytes(uint32_t n_blocks, uint32_t block_size, int level) {
    return (size_t)enc_full_warps(n_blocks) * enc_layout(block_size, level).total;
}

extern "C" uint32_t zxg_ps_stage_stride(uint32_t block_size) { return enc_staging_stride(block_size); }

extern "C" int zxg_ps_decode(const zxc_b200_job_t* h_jobs, uint32_t n, zxc_b200_job_t* d_jobs, int32_t* d_status,
                             void* d_dst, void* d_scratch, size_t scratch_size, unsigned long long* d_counter,
                             uint32_t block_size, int verify, int32_t* h_status, void* stream) {
    cudaStream_t st = (cudaStream_t)stream;
    int rc = ps_cuda(cudaMemcpyAsync(d_jobs, h_jobs, (size_t)n * sizeof(zxc_b200_job_t), cudaMemcpyHostToDevice, st));
    /* the jobs' offsets are device addresses: the decode's source base is zero */
    if (rc == ZXC_OK)
        rc = launch_decode(NULL, d_dst, d_jobs, n, d_status, NULL, 0, NULL, d_scratch, scratch_size, block_size, verify,
                           d_counter, st, 0);
    if (rc == ZXC_OK) rc = ps_cuda(cudaMemcpyAsync(h_status, d_status, (size_t)n * 4, cudaMemcpyDeviceToHost, st));
    if (rc == ZXC_OK) rc = ps_cuda(cudaStreamSynchronize(st));
    return rc;
}

extern "C" int zxg_ps_encode(const void* d_src, uint64_t src_size, uint32_t block_size, int level, int checksum,
                             uint32_t n_blocks, void* d_stage, uint32_t* d_st, void* d_scratch,
                             unsigned long long* d_counter, uint32_t* h_st, void* stream) {
    cudaStream_t st = (cudaStream_t)stream;
    const EncLaunch E = {(const u8*)d_src, src_size, block_size, n_blocks, level, checksum, (u8*)d_stage, d_st,
                         (u8*)d_scratch, enc_full_warps(n_blocks), d_counter, NULL, NULL, 0, NULL};
    int rc = launch_encode(E, st);
    if (rc != ZXC_OK) return rc;
    zxc_ps_trailers<<<(n_blocks + 255) / 256, 256, 0, st>>>((const u8*)d_stage, enc_staging_stride(block_size), d_st,
                                                            d_st + n_blocks, n_blocks);
    __atomic_add_fetch(&g_launches, 1, __ATOMIC_RELAXED);
    rc = ps_cuda(cudaGetLastError());
    if (rc == ZXC_OK) rc = ps_cuda(cudaMemcpyAsync(h_st, d_st, (size_t)n_blocks * 8, cudaMemcpyDeviceToHost, st));
    if (rc == ZXC_OK) rc = ps_cuda(cudaStreamSynchronize(st));
    return rc;
}

extern "C" int zxg_ps_gather(const zxg_psseg_t* h_segs, uint32_t n, zxg_psseg_t* d_segs, void* stream) {
    if (n == 0) return ZXC_OK;
    cudaStream_t st = (cudaStream_t)stream;
    int rc = ps_cuda(cudaMemcpyAsync(d_segs, h_segs, (size_t)n * sizeof *h_segs, cudaMemcpyHostToDevice, st));
    if (rc != ZXC_OK) return rc;
    const u32 gmax = (u32)(g_sm_count > 0 ? g_sm_count : 132) * 8u;
    zxc_ps_gather<<<n < gmax ? n : gmax, 256, 0, st>>>(d_segs, n);
    __atomic_add_fetch(&g_launches, 1, __ATOMIC_RELAXED);
    return ps_cuda(cudaGetLastError());
}

/* ------------------------------------------------------------------------- */
/* random access into a seekable frame in HBM                                */
/* (zxc_b200_seekable_device_*: zxc_dseek.c drives these, kernels in         */
/* zxc_dseek.cuh)                                                            */
/* ------------------------------------------------------------------------- */
extern "C" int zxg_d2h_sync(void* h_dst, const void* d_src, size_t bytes, void* stream) {
    cudaStream_t st = (cudaStream_t)stream;
    if (cudaMemcpyAsync(h_dst, d_src, bytes, cudaMemcpyDeviceToHost, st) != cudaSuccess ||
        cudaStreamSynchronize(st) != cudaSuccess) {
        cudaGetLastError();
        return ZXC_B200_ERROR_CUDA;
    }
    return ZXC_OK;
}

extern "C" int zxg_h2d_sync(void* d_dst, const void* h_src, size_t bytes, void* stream) {
    cudaStream_t st = (cudaStream_t)stream;
    if (cudaMemcpyAsync(d_dst, h_src, bytes, cudaMemcpyHostToDevice, st) != cudaSuccess ||
        cudaStreamSynchronize(st) != cudaSuccess) {
        cudaGetLastError();
        return ZXC_B200_ERROR_CUDA;
    }
    return ZXC_OK;
}

extern "C" const void* zxg_host_mapped(const void* h, size_t bytes) {
    /* both ends of the frame: page-locked (cudaHostAlloc, or cudaHostRegister of a range that holds it), mapped for the
     * current device, and one mapping */
    cudaPointerAttributes a0, a1;
    const u8* end = (const u8*)h + bytes - 1;
    if (cudaPointerGetAttributes(&a0, h) != cudaSuccess || cudaPointerGetAttributes(&a1, end) != cudaSuccess) {
        cudaGetLastError();
        return NULL;
    }
    if (a0.type != cudaMemoryTypeHost || a1.type != cudaMemoryTypeHost || !a0.devicePointer || !a1.devicePointer ||
        (const u8*)a1.devicePointer - (const u8*)a0.devicePointer != (ptrdiff_t)(bytes - 1))
        return NULL;
    return a0.devicePointer;
}

extern "C" void* zxg_dev_alloc(size_t bytes) {
    void* d = NULL;
    if (cudaMalloc(&d, bytes) != cudaSuccess) {
        cudaGetLastError();
        return NULL;
    }
    return d;
}

extern "C" void zxg_dev_free(void* d) {
    if (!d) return;
    cudaDeviceSynchronize(); /* range calls still in flight on any stream may read it */
    cudaFree(d);
}

/* ---- prepared dictionaries (zxc_b200_dict_device: zxc_api.c): the decode region, then the encode region ---- */
static size_t ddict_enc_off(u32 dict_size) { return r256((size_t)dict_size + ZXC_HUF_TABLE_SIZE); }

extern "C" size_t zxg_ddict_bytes(uint32_t dict_size) { return ddict_enc_off(dict_size) + enc_dict_bytes(dict_size, 2); }

extern "C" int zxg_ddict_build(void* d_base, const void* h_dict, uint32_t dict_size, const void* h_dec_huf,
                               const uint8_t* h_lens, void* stream, zxg_ddict_t* dd) {
    cudaStream_t st = (cudaStream_t)stream;
    u8* base = (u8*)d_base;
    u8* enc = base + ddict_enc_off(dict_size);
    static const int seed_levels[2] = {1, 3}; /* hash5 off, on */
    int rc = dec_build_dict(base, h_dict, dict_size, h_dec_huf, st);
    if (rc == ZXC_OK) rc = enc_build_dict(enc, h_dict, dict_size, seed_levels, 2, h_lens, st);
    if (rc == ZXC_OK && cudaStreamSynchronize(st) != cudaSuccess) rc = ZXC_B200_ERROR_CUDA;
    if (rc != ZXC_OK) {
        cudaGetLastError();
        return rc;
    }
    dd->dec = base;
    dd->dec_huf = h_dec_huf ? base + dict_size : NULL;
    dd->enc = enc;
    dd->enc_lens = h_lens ? enc + enc_dict_pad(dict_size) + 2 * ENC_SEED_PAIR : NULL;
    dd->dict_size = dict_size;
    return ZXC_OK;
}

/* Scratch layout, from the caller's base rounded up to 256 bytes (every region 256-aligned):
 *   DSeekState | per-range records (n) | tile sums | slot table (2n jobs, 2n status) | direct table (J jobs, J status) |
 *   slots (2n x round_up(block_size, 16)) | decode scratch (per-warp regions, deferred list)
 * The decode scratch holds the per-warp regions of the larger of the two decode launches, grid_for(max(J, 2n)) warps,
 * so a call with few ranges and few blocks needs no more than its launches use.  total grows with J, and the call
 * takes the largest J whose layout fits the scratch it is given.
 * A frame in host memory adds the staged-size tile sums behind the tile sums and the staging area behind the slots:
 * (J + 2n) x max_comp + DS_STAGE_RANGE n bytes.  A range admitted by the job table stages its nd + ns blocks of at most
 * max_comp bytes each, plus a skew below 16, DS_STAGE_PAD and rounding to 16 (at most 38 bytes), and the admitted
 * ranges hold at most J direct and 2n slot jobs: the staging area never decides which ranges are admitted. */
struct DSeekLayout {
    size_t recs, tiles, ptiles, sjobs, sstatus, djobs, dstatus, slots, stage, dec, dec_bytes, total;
    u32 J, stride;
};
#define DS_J_MAX 0x7FFFFFFFu
#define DS_RANGES_MAX (1u << 30) /* the slot table's 2n entries stay below 2^31 */
#define DS_STAGE_RANGE 48u

static void ds_layout(u32 bs, u32 n, u32 J, u32 max_comp, DSeekLayout* L) {
    size_t o = DS_STATE_BYTES;
    L->recs = o;
    o += r256((size_t)n * sizeof(DSeekRec));
    L->tiles = o;
    o += r256(((size_t)n + ASM_TILE - 1) / ASM_TILE * 16);
    L->ptiles = o;
    if (max_comp) o += r256(((size_t)n + ASM_TILE - 1) / ASM_TILE * 8);
    L->sjobs = o;
    o += r256((size_t)2 * n * sizeof(zxc_b200_job_t));
    L->sstatus = o;
    o += r256((size_t)2 * n * 4);
    L->djobs = o;
    o += r256((size_t)J * sizeof(zxc_b200_job_t));
    L->dstatus = o;
    o += r256((size_t)J * 4);
    L->stride = (bs + 15u) & ~15u;
    L->slots = o;
    o += r256((size_t)2 * n * L->stride);
    L->stage = o;
    L->J = J;
    if (max_comp && ((size_t)J + 2ull * n) > (SIZE_MAX >> 2) / max_comp) { /* a size no scratch has */
        L->total = SIZE_MAX;
        return;
    }
    if (max_comp) o += r256(((size_t)J + 2ull * n) * max_comp + (size_t)DS_STAGE_RANGE * n);
    L->dec = o;
    L->dec_bytes = launch_scratch_bytes(J > 2 * n ? J : 2 * n, bs);
    L->total = o + L->dec_bytes + 256; /* base alignment slack */
}

extern "C" size_t zxg_dseek_scratch_bytes(uint32_t block_size, uint32_t n_ranges, uint64_t J, uint32_t max_comp) {
    if (zxg_init() != ZXC_OK || J > DS_J_MAX || n_ranges > DS_RANGES_MAX) return 0;
    DSeekLayout L;
    ds_layout(block_size, n_ranges, J < 1 ? 1u : (u32)J, max_comp, &L);
    return L.total == SIZE_MAX ? 0 : L.total;
}

extern "C" int zxg_dseek_ranges(const zxg_dseek_t* h, const zxc_b200_range_t* d_ranges, uint32_t n_ranges, void* d_dst,
                                uint64_t dst_capacity, void* d_scratch, size_t scratch_size, int64_t* d_results,
                                void* stream) {
    const u32 bs = h->block_size, n = n_ranges, mc = h->max_comp;
    const bool host = mc != 0;
    if (n > DS_RANGES_MAX) return ZXC_ERROR_MEMORY;
    DSeekLayout L;
    ds_layout(bs, n, 1, mc, &L);
    if (L.total > scratch_size) return ZXC_ERROR_MEMORY;
    /* the largest direct table whose layout fits: L.total grows with J */
    ds_layout(bs, n, (u32)largest_fit(1, DS_J_MAX, [&](u64 J) {
                  ds_layout(bs, n, (u32)J, mc, &L);
                  return L.total <= scratch_size;
              }),
              mc, &L);
    cudaStream_t st = (cudaStream_t)stream;
    u8* base = (u8*)(((uintptr_t)d_scratch + 255) & ~(uintptr_t)255);
    DSeekState* S = (DSeekState*)base;
    const bool has_dict = h->d_dict && h->dict_size;
    DSeekArgs A;
    A.offs = (const unsigned long long*)h->d_offs;
    A.ranges = d_ranges;
    A.dst = (u8*)d_dst;
    A.slots = base + L.slots;
    A.results = (long long*)d_results;
    A.st = S;
    A.recs = (DSeekRec*)(base + L.recs);
    A.tiles = (unsigned long long*)(base + L.tiles);
    A.djobs = (zxc_b200_job_t*)(base + L.djobs);
    A.dstatus = (i32*)(base + L.dstatus);
    A.sjobs = (zxc_b200_job_t*)(base + L.sjobs);
    A.sstatus = (i32*)(base + L.sstatus);
    A.total = h->total;
    A.dst_capacity = dst_capacity;
    A.n = n;
    A.J = L.J;
    A.block_size = bs;
    A.slot_stride = L.stride;
    A.need_dict = h->dict_id != 0 && !has_dict;
    A.hsrc = host ? (const u8*)h->d_src : NULL;
    A.stage = host ? base + L.stage : NULL;
    A.ptiles = host ? (unsigned long long*)(base + L.ptiles) : NULL;
    A.src_size = h->src_size;
    const u32 n_tiles = (n + ASM_TILE - 1) / ASM_TILE;
    /* a warp per range, and enough threads to zero the status words in front of both tables quickly */
    const u64 by_ranges = ((u64)n * 32 + DS_THREADS - 1) / DS_THREADS;
    u64 by_zero = ((u64)L.J + 2ull * n + DS_THREADS * 16 - 1) / (DS_THREADS * 16);
    if (by_zero > 4096) by_zero = 4096;
    const u32 emit_grid = (u32)(by_ranges > by_zero ? by_ranges : by_zero);
    if (host) {
        /* the same plan with staged sources, then the admitted ranges' spans over PCIe: a grid the SMs hold at once */
        zxc_dseek_tiles_host<<<n_tiles, ASM_THREADS, 0, st>>>(A);
        zxc_dseek_scan_host<<<1, ASM_SCAN_THREADS, 0, st>>>(A);
        zxc_dseek_emit_host<<<emit_grid, DS_THREADS, 0, st>>>(A);
        zxc_dseek_fetch<<<(u32)(g_sm_count > 0 ? g_sm_count : 132) * 8u, DS_FETCH_THREADS, 0, st>>>(A);
        __atomic_add_fetch(&g_launches, 4, __ATOMIC_RELAXED);
    } else {
        zxc_dseek_tiles<<<n_tiles, ASM_THREADS, 0, st>>>(A);
        zxc_dseek_scan<<<1, ASM_SCAN_THREADS, 0, st>>>(A);
        zxc_dseek_emit<<<emit_grid, DS_THREADS, 0, st>>>(A);
        __atomic_add_fetch(&g_launches, 3, __ATOMIC_RELAXED);
    }
    if (cudaGetLastError() != cudaSuccess) return ZXC_B200_ERROR_CUDA;
    /* the blocks covered whole, in place; then the partly covered ones into their slots.  Stream order lets the two
     * runs share the per-warp scratch and the deferred list; each has its own counters. */
    u8* dec = base + L.dec;
    const void* dict = has_dict ? h->d_dict : NULL;
    const void* huf = has_dict ? h->d_dict_huf : NULL;
    const void* src = host ? (const void*)A.stage : h->d_src;
    int rc = launch_decode(src, d_dst, A.djobs, L.J, A.dstatus, dict, h->dict_size, huf, dec, L.dec_bytes, bs, 0,
                           S->ctr[0], st, 1);
    if (rc != ZXC_OK) return rc;
    rc = launch_decode(src, A.slots, A.sjobs, 2 * n, A.sstatus, dict, h->dict_size, huf, dec, L.dec_bytes, bs, 0,
                       S->ctr[1], st, 1);
    if (rc != ZXC_OK) return rc;
    zxc_dseek_finish<<<n, DS_THREADS, 0, st>>>(A);
    __atomic_add_fetch(&g_launches, 1, __ATOMIC_RELAXED);
    return cudaGetLastError() == cudaSuccess ? ZXC_OK : ZXC_B200_ERROR_CUDA;
}

/* ------------------------------------------------------------------------- */
/* a SEK table for a device-resident frame (zxc_b200_add_seek_table_device:  */
/* kernels in zxc_dindex.cuh)                                                */
/* ------------------------------------------------------------------------- */
/* Scratch layout, every region 256-aligned but the last: the state (DI_STATE_BYTES) | the scan tiles' counts (u64 per
 * DI_TILE frame offsets) | C candidate offsets (u64) | their sizes (u32) | two jump tables (C x u32) | the marks (C
 * bytes) | the mark tiles (u64 per ASM_TILE candidates) | the plan (J x zxc_b200_job_t), not rounded, so that the
 * size grows with every block and the call finds J back from scratch_size.  C = 2 J + DI_C_SLACK. */
#define DI_C_SLACK 1024u
#define DI_J_MAX (1u << 28)
struct DIdxLayout {
    size_t tiles, off, len, jump[2], mark, mtiles, plan, total;
    u32 C, J, n_tiles;
};
static bool di_layout(uint64_t frame_size, uint64_t J, DIdxLayout* L) {
    const u64 scan = frame_size > ZXC_FILE_FOOTER_SIZE + ZXF_BLOCK_HDR ? frame_size - ZXC_FILE_FOOTER_SIZE - ZXF_BLOCK_HDR
                                                                         : 1; /* offsets 0 .. the last header's */
    const u64 n_tiles = (scan + 1 + DI_TILE - 1) / DI_TILE;
    if (J > DI_J_MAX || n_tiles > 0x7FFFFFFFull) return false;
    const u64 C = 2 * J + DI_C_SLACK;
    size_t o = DI_STATE_BYTES;
    L->tiles = o;
    o += r256((size_t)n_tiles * 8);
    L->off = o;
    o += r256((size_t)C * 8);
    L->len = o;
    o += r256((size_t)C * 4);
    for (int t = 0; t < 2; t++) {
        L->jump[t] = o;
        o += r256((size_t)C * 4);
    }
    L->mark = o;
    o += r256((size_t)C);
    L->mtiles = o;
    o += r256((size_t)(C + ASM_TILE - 1) / ASM_TILE * 8);
    L->plan = o;
    o += (size_t)J * sizeof(zxc_b200_job_t);
    L->total = o + 256; /* base alignment slack */
    L->C = (u32)C;
    L->J = (u32)J;
    L->n_tiles = (u32)n_tiles;
    return true;
}

extern "C" size_t zxg_seek_table_scratch_bytes(uint64_t frame_size, uint32_t max_blocks) {
    if (zxg_init() != ZXC_OK) return 0;
    DIdxLayout L;
    return di_layout(frame_size, max_blocks, &L) ? L.total : 0;
}

/* a grid-stride kernel's CTAs for n items */
static u32 di_grid(u64 n) {
    const u64 g = (n + DI_THREADS - 1) / DI_THREADS;
    return g < 1 ? 1u : (g > DI_GRID_MAX ? (u32)DI_GRID_MAX : (u32)g);
}

extern "C" int zxg_add_seek_table_device(void* d_buffer, uint64_t frame_size, uint64_t buffer_capacity,
                                         void* d_scratch, size_t scratch_size, int64_t* d_result, void* stream) {
    const int irc = zxg_init();
    if (irc != ZXC_OK) return irc;
    DIdxLayout L;
    if (!di_layout(frame_size, 0, &L) || L.total > scratch_size) return ZXC_ERROR_MEMORY;
    /* the largest plan whose layout fits: L.total grows with J */
    di_layout(frame_size, largest_fit(0, DI_J_MAX, [&](u64 J) { return di_layout(frame_size, J, &L) && L.total <= scratch_size; }),
              &L);
    cudaStream_t st = (cudaStream_t)stream;
    u8* base = (u8*)(((uintptr_t)d_scratch + 255) & ~(uintptr_t)255);
    DIdxArgs A;
    A.buf = (u8*)d_buffer;
    A.size = frame_size;
    A.cap = buffer_capacity;
    A.st = (DIdxState*)base;
    A.tiles = (unsigned long long*)(base + L.tiles);
    A.off = (unsigned long long*)(base + L.off);
    A.len = (unsigned int*)(base + L.len);
    A.jump[0] = (unsigned int*)(base + L.jump[0]);
    A.jump[1] = (unsigned int*)(base + L.jump[1]);
    A.mark = base + L.mark;
    A.mtiles = (unsigned long long*)(base + L.mtiles);
    A.plan = (zxc_b200_job_t*)(base + L.plan);
    A.result = (long long*)d_result;
    A.C = L.C;
    A.J = L.J;
    A.n_tiles = L.n_tiles;
    const u32 by_cand = di_grid(L.C), by_plan = di_grid(L.J);
    const u32 m_tiles = (L.C + ASM_TILE - 1) / ASM_TILE;
    zxc_dindex_probe<<<1, 1, 0, st>>>(A);
    zxc_dindex_count<<<L.n_tiles, DI_THREADS, 0, st>>>(A);
    zxc_dindex_tscan<<<1, ASM_SCAN_THREADS, 0, st>>>(A);
    zxc_dindex_emit<<<L.n_tiles, DI_THREADS, 0, st>>>(A);
    zxc_dindex_links<<<by_cand, DI_THREADS, 0, st>>>(A);
    for (u32 r = 0; r < DI_ROUNDS; r++) zxc_dindex_round<<<by_cand, DI_THREADS, 0, st>>>(A, r);
    zxc_dindex_mtiles<<<m_tiles, ASM_THREADS, 0, st>>>(A);
    zxc_dindex_mscan<<<1, ASM_SCAN_THREADS, 0, st>>>(A);
    zxc_dindex_memit<<<m_tiles, ASM_THREADS, 0, st>>>(A);
    zxc_dindex_prove<<<by_plan, DI_THREADS, 0, st>>>(A);
    zxc_dindex_walk<<<1, 32, 0, st>>>(A);
    zxc_dindex_check<<<by_plan, DI_THREADS, 0, st>>>(A);
    zxc_dindex_decide<<<1, 1, 0, st>>>(A);
    zxc_dindex_write<<<by_plan, DI_THREADS, 0, st>>>(A);
    __atomic_add_fetch(&g_launches, 13 + DI_ROUNDS, __ATOMIC_RELAXED);
    return cudaGetLastError() == cudaSuccess ? ZXC_OK : ZXC_B200_ERROR_CUDA;
}

/* ------------------------------------------------------------------------- */
/* dictionary training (zxc_train.c drives these; kernels in zxc_train.cuh)   */
/* ------------------------------------------------------------------------- */
static_assert(sizeof(TrainSeg) == sizeof(zxg_seg_t), "TrainSeg and zxg_seg_t are the same record");

static __thread double t_train_ms[ZXG_T_N];
extern "C" double* zxg_train_times(void) { return t_train_ms; }

/* Packs n host pieces back to back into d_dst through the context's pinned bounce buffers: one DMA per 32 MiB, not
 * one per piece (a million 100-byte samples is an ordinary training input).  A NULL piece of non-zero size reads as
 * zeros. */
static int h2d_gather(zxg_ctx* c, u8* d_dst, const void* const* pieces, const size_t* sizes, size_t n) {
    const int rc = ensure_pins(c);
    if (rc != ZXC_OK) return rc;
    size_t fill = 0, d_off = 0;
    int slot = 0;
    cudaEventSynchronize(c->pin_ev[slot]);
    for (size_t i = 0; i < n; i++) {
        const u8* s = (const u8*)pieces[i];
        size_t left = sizes[i];
        while (left) {
            const size_t take = left < PIN_CHUNK - fill ? left : PIN_CHUNK - fill;
            if (s) {
                pool_memcpy(c->device, (u8*)c->pin[slot] + fill, s, take);
                s += take;
            } else {
                memset((u8*)c->pin[slot] + fill, 0, take);
            }
            fill += take;
            left -= take;
            if (fill == PIN_CHUNK) {
                if (cudaMemcpyAsync(d_dst + d_off, c->pin[slot], fill, cudaMemcpyHostToDevice, c->stream) != cudaSuccess)
                    return ZXC_B200_ERROR_CUDA;
                cudaEventRecord(c->pin_ev[slot], c->stream);
                d_off += fill;
                fill = 0;
                slot ^= 1;
                cudaEventSynchronize(c->pin_ev[slot]); /* the previous use of this bounce buffer */
            }
        }
    }
    if (fill) {
        if (cudaMemcpyAsync(d_dst + d_off, c->pin[slot], fill, cudaMemcpyHostToDevice, c->stream) != cudaSuccess)
            return ZXC_B200_ERROR_CUDA;
        cudaEventRecord(c->pin_ev[slot], c->stream);
    }
    return ZXC_OK;
}

struct train_events {
    cudaEvent_t ev[8];
    int n;
};
static int tev_init(train_events* T, int n) {
    T->n = 0;
    for (int i = 0; i < n; i++) {
        if (cudaEventCreate(&T->ev[i]) != cudaSuccess) return ZXC_B200_ERROR_CUDA;
        T->n++;
    }
    return ZXC_OK;
}
static double tev_ms(train_events* T, int a, int b) {
    float ms = 0;
    cudaEventElapsedTime(&ms, T->ev[a], T->ev[b]);
    return ms;
}
static void tev_free(train_events* T) {
    for (int i = 0; i < T->n; i++) cudaEventDestroy(T->ev[i]);
}

/* Packs n device pieces back to back into d_dst in one zxc_ps_gather launch (none when they hold no bytes).  The host
 * cuts every piece into parts of at most ZXG_PS_PIECE bytes and uploads that table into ZXG_BUF_OUT, which no trainer
 * uses otherwise.  A NULL piece of non-zero size reads as zeros. */
static int d2d_gather(zxg_ctx* c, u8* d_dst, const void* const* pieces, const size_t* sizes, size_t n) {
    size_t m = 0;
    for (size_t i = 0; i < n; i++) m += (sizes[i] + ZXG_PS_PIECE - 1) / ZXG_PS_PIECE;
    if (m == 0) return ZXC_OK;
    if (m > UINT32_MAX) return ZXC_ERROR_MEMORY;
    zxg_psseg_t* h = (zxg_psseg_t*)malloc(m * sizeof *h);
    zxg_psseg_t* d = (zxg_psseg_t*)zxg_buffer(c, ZXG_BUF_OUT, m * sizeof *h);
    if (!h || !d) {
        free(h);
        return ZXC_ERROR_MEMORY;
    }
    u64 off = 0;
    size_t k = 0;
    for (size_t i = 0; i < n; i++) {
        const u64 s = (u64)(uintptr_t)pieces[i];
        for (u64 o = 0; o < sizes[i]; o += ZXG_PS_PIECE, k++) {
            h[k].src = s ? s + o : 0;
            h[k].dst = (u64)(uintptr_t)(d_dst + off + o);
            h[k].len = sizes[i] - o < ZXG_PS_PIECE ? sizes[i] - o : ZXG_PS_PIECE;
        }
        off += sizes[i];
    }
    int rc = zxg_h2d(c, d, h, m * sizeof *h); /* the host table has been read when it returns */
    free(h);
    if (rc != ZXC_OK) return rc;
    const u32 gmax = (u32)(g_sm_count > 0 ? g_sm_count : 132) * 8u;
    zxc_ps_gather<<<m < gmax ? (u32)m : gmax, 256, 0, c->stream>>>(d, (u32)m);
    __atomic_add_fetch(&g_launches, 1, __ATOMIC_RELAXED);
    return cudaGetLastError() == cudaSuccess ? ZXC_OK : ZXC_B200_ERROR_CUDA;
}

/* Fills d_dst with the samples, packed: from host memory through the bounce buffers, or, for device samples, after the
 * work enqueued on the caller's stream (an event orders the context's stream behind it) by d2d_gather.  T->ev[0] is
 * recorded once the context's stream may start, so the upload slot times the transfer alone. */
static int gather_samples(zxg_ctx* c, u8* d_dst, const void* const* pieces, const size_t* sizes, size_t n,
                          const zxg_train_src_t* src, train_events* T) {
    if (src && src->device) {
        cudaEvent_t ev;
        if (cudaEventCreateWithFlags(&ev, cudaEventDisableTiming) != cudaSuccess) return ZXC_B200_ERROR_CUDA;
        const bool ok = cudaEventRecord(ev, (cudaStream_t)src->stream) == cudaSuccess &&
                        cudaStreamWaitEvent(c->stream, ev, 0) == cudaSuccess;
        cudaEventDestroy(ev);
        if (!ok) return ZXC_B200_ERROR_CUDA;
        cudaEventRecord(T->ev[0], c->stream);
        return d2d_gather(c, d_dst, pieces, sizes, n);
    }
    cudaEventRecord(T->ev[0], c->stream);
    return h2d_gather(c, d_dst, pieces, sizes, n);
}

static int grid_cap(unsigned long long want, u32 per_sm) {
    const unsigned long long cap = (unsigned long long)(g_sm_count > 0 ? g_sm_count : 132) * per_sm;
    return (int)(want < 1 ? 1 : (want < cap ? want : cap));
}

/* device layout of the content trainer, behind the corpus: ZXG_BUF_AUX = [freq u32 x 65536 | result words | starts |
 * kept segments]; ZXG_BUF_JOBS = [ordered segments | hash offsets | chunk starts | picks | output] */
#define TRN_RES_OFF ((size_t)TRN_HASH_SIZE * 4)
#define TRN_STARTS_OFF (TRN_RES_OFF + 256)
static size_t trn_kept_off(u32 n_starts) { return (TRN_STARTS_OFF + (size_t)n_starts * sizeof(TrainSeg) + 255) & ~(size_t)255; }

extern "C" int zxg_train_segments(zxg_ctx* c, const void* const* samples, const size_t* sizes, size_t n_samples,
                                  uint64_t corpus_size, uint64_t freq_stride, uint64_t seg_stride, uint32_t n_starts,
                                  uint32_t seg_alloc, zxg_seg_t* h_segs, uint32_t* n_segs, const zxg_train_src_t* src) {
    *n_segs = 0;
    u8* d_corpus = (u8*)zxg_buffer(c, ZXG_BUF_IN, (size_t)corpus_size + 16);
    u8* aux = (u8*)zxg_buffer(c, ZXG_BUF_AUX, trn_kept_off(n_starts) + (size_t)seg_alloc * sizeof(TrainSeg) + 256);
    if (!d_corpus || !aux) return ZXC_ERROR_MEMORY;
    u32* d_freq = (u32*)aux;
    u32* d_res = (u32*)(aux + TRN_RES_OFF);
    TrainSeg* d_starts = (TrainSeg*)(aux + TRN_STARTS_OFF);
    TrainSeg* d_kept = (TrainSeg*)(aux + trn_kept_off(n_starts));
    train_events T;
    int rc = tev_init(&T, 4);
    if (rc == ZXC_OK) rc = gather_samples(c, d_corpus, samples, sizes, n_samples, src, &T);
    if (rc == ZXC_OK && (cudaMemsetAsync(d_corpus + corpus_size, 0, 16, c->stream) != cudaSuccess ||
                         cudaMemsetAsync(d_freq, 0, TRN_RES_OFF + 256, c->stream) != cudaSuccess))
        rc = ZXC_B200_ERROR_CUDA;
    if (rc == ZXC_OK) {
        cudaEventRecord(T.ev[1], c->stream);
        const unsigned long long kgram_limit = corpus_size - TRN_K + 1;
        const unsigned long long n_count = (kgram_limit + freq_stride - 1) / freq_stride;
        zxc_train_count_kernel<<<grid_cap((n_count + 255) / 256, 16), 256, 0, c->stream>>>(d_corpus, kgram_limit, freq_stride,
                                                                                          d_freq);
        cudaEventRecord(T.ev[2], c->stream);
        if (cudaFuncSetAttribute(zxc_train_seg_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, TRN_SEG_SMEM) != cudaSuccess)
            rc = ZXC_B200_ERROR_CUDA;
    }
    if (rc == ZXC_OK) {
        zxc_train_seg_kernel<<<grid_cap(((unsigned long long)n_starts + 31) / 32, 1), TRN_CTA, TRN_SEG_SMEM, c->stream>>>(
            d_corpus, corpus_size, seg_stride, n_starts, d_freq, d_starts);
        zxc_train_compact_kernel<<<1, TRN_CTA, 0, c->stream>>>(d_starts, n_starts, seg_alloc, d_kept, d_res);
        __atomic_add_fetch(&g_launches, 3, __ATOMIC_RELAXED);
        cudaEventRecord(T.ev[3], c->stream);
        u32 n = 0;
        if (cudaMemcpyAsync(&n, d_res, 4, cudaMemcpyDeviceToHost, c->stream) != cudaSuccess ||
            cudaStreamSynchronize(c->stream) != cudaSuccess)
            rc = ZXC_B200_ERROR_CUDA;
        else if (n && (cudaMemcpyAsync(h_segs, d_kept, (size_t)n * sizeof(TrainSeg), cudaMemcpyDeviceToHost, c->stream) != cudaSuccess ||
                       cudaStreamSynchronize(c->stream) != cudaSuccess))
            rc = ZXC_B200_ERROR_CUDA;
        *n_segs = n;
    }
    if (rc == ZXC_OK) {
        t_train_ms[ZXG_T_UPLOAD] = tev_ms(&T, 0, 1);
        t_train_ms[ZXG_T_COUNT] = tev_ms(&T, 1, 2);
        t_train_ms[ZXG_T_SEGMENTS] = tev_ms(&T, 2, 3);
    } else {
        fprintf(stderr, "libzxc (CUDA build): dictionary training failed: %s\n", cudaGetErrorString(cudaGetLastError()));
    }
    tev_free(&T);
    return rc;
}

extern "C" int zxg_train_pick(zxg_ctx* c, uint64_t corpus_size, const zxg_seg_t* h_sorted, uint32_t n_segs, uint32_t capacity,
                              uint8_t* h_out, uint32_t* filled) {
    *filled = 0;
    if (n_segs == 0) return ZXC_OK;
    /* hash offsets in pick order, and the chunks of at most TRN_CHUNK hashes the pick stages at a time */
    u32* h_idx = (u32*)malloc(((size_t)n_segs + 1) * 2 * sizeof(u32));
    if (!h_idx) return ZXC_ERROR_MEMORY;
    u32* hoff = h_idx;
    u32* chunk_first = h_idx + n_segs + 1;
    u32 n_chunks = 0, acc = 0;
    for (u32 j = 0; j < n_segs; j++) {
        const u32 nk = h_sorted[j].len / TRN_K;
        if (j == 0 || acc - hoff[chunk_first[n_chunks - 1]] + nk > TRN_CHUNK) chunk_first[n_chunks++] = j;
        hoff[j] = acc;
        acc += nk;
    }
    hoff[n_segs] = acc;
    chunk_first[n_chunks] = n_segs;
    const size_t o_hoff = ((size_t)n_segs * sizeof(TrainSeg) + 255) & ~(size_t)255;
    const size_t o_chunk = (o_hoff + ((size_t)n_segs + 1) * 4 + 255) & ~(size_t)255;
    const size_t o_picks = (o_chunk + ((size_t)n_chunks + 1) * 4 + 255) & ~(size_t)255;
    const size_t o_out = (o_picks + (size_t)n_segs * sizeof(TrainPick) + 255) & ~(size_t)255;
    u8* jb = (u8*)zxg_buffer(c, ZXG_BUF_JOBS, o_out + 65536 + 16);
    unsigned short* d_hash = (unsigned short*)zxg_buffer(c, ZXG_BUF_SCRATCH, (size_t)acc * 2 + 16);
    const u8* d_corpus = (const u8*)zxg_buffer(c, ZXG_BUF_IN, (size_t)corpus_size + 16);
    u8* aux = (u8*)c->buf[ZXG_BUF_AUX];
    if (!jb || !d_hash || !d_corpus || !aux) {
        free(h_idx);
        return ZXC_ERROR_MEMORY;
    }
    TrainSeg* d_seg = (TrainSeg*)jb;
    u32* d_hoff = (u32*)(jb + o_hoff);
    u32* d_chunk = (u32*)(jb + o_chunk);
    TrainPick* d_picks = (TrainPick*)(jb + o_picks);
    u8* d_out = jb + o_out;
    u32* d_res = (u32*)(aux + TRN_RES_OFF) + 4;
    train_events T;
    int rc = tev_init(&T, 2);
    if (rc == ZXC_OK &&
        (cudaMemcpyAsync(d_seg, h_sorted, (size_t)n_segs * sizeof(TrainSeg), cudaMemcpyHostToDevice, c->stream) != cudaSuccess ||
         cudaMemcpyAsync(d_hoff, hoff, ((size_t)n_segs + 1) * 4, cudaMemcpyHostToDevice, c->stream) != cudaSuccess ||
         cudaMemcpyAsync(d_chunk, chunk_first, ((size_t)n_chunks + 1) * 4, cudaMemcpyHostToDevice, c->stream) != cudaSuccess ||
         cudaFuncSetAttribute(zxc_train_pick_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, TRN_PICK_SMEM) != cudaSuccess))
        rc = ZXC_B200_ERROR_CUDA;
    u32 res[2] = {0, 0};
    if (rc == ZXC_OK) {
        cudaEventRecord(T.ev[0], c->stream);
        zxc_train_hash_kernel<<<grid_cap(((unsigned long long)n_segs + 7) / 8, 8), 256, 0, c->stream>>>(d_corpus, d_seg, d_hoff,
                                                                                                     n_segs, d_hash);
        zxc_train_pick_kernel<<<1, TRN_CTA, TRN_PICK_SMEM, c->stream>>>(d_seg, d_hoff, d_hash, d_chunk, n_chunks, (const u32*)aux,
                                                                        capacity, d_picks, d_res);
        __atomic_add_fetch(&g_launches, 2, __ATOMIC_RELAXED);
        cudaEventRecord(T.ev[1], c->stream);
        if (cudaMemcpyAsync(res, d_res, 8, cudaMemcpyDeviceToHost, c->stream) != cudaSuccess ||
            cudaStreamSynchronize(c->stream) != cudaSuccess)
            rc = ZXC_B200_ERROR_CUDA;
    }
    if (rc == ZXC_OK && res[0]) {
        zxc_train_emit_kernel<<<grid_cap(((unsigned long long)res[0] + 7) / 8, 8), 256, 0, c->stream>>>(d_corpus, d_picks, res[0],
                                                                                                      res[1], d_out);
        __atomic_add_fetch(&g_launches, 1, __ATOMIC_RELAXED);
        if (cudaMemcpyAsync(h_out, d_out, res[1], cudaMemcpyDeviceToHost, c->stream) != cudaSuccess ||
            cudaStreamSynchronize(c->stream) != cudaSuccess)
            rc = ZXC_B200_ERROR_CUDA;
    }
    if (rc == ZXC_OK) {
        t_train_ms[ZXG_T_PICK] = tev_ms(&T, 0, 1);
        *filled = res[1];
    } else {
        fprintf(stderr, "libzxc (CUDA build): dictionary training failed: %s\n", cudaGetErrorString(cudaGetLastError()));
    }
    tev_free(&T);
    free(h_idx);
    return rc;
}

extern "C" int zxg_train_tail(zxg_ctx* c, uint64_t corpus_size, uint32_t bytes, uint8_t* h_out) {
    const u8* d_corpus = (const u8*)zxg_buffer(c, ZXG_BUF_IN, (size_t)corpus_size + 16);
    if (!d_corpus) return ZXC_ERROR_MEMORY;
    if (cudaMemcpyAsync(h_out, d_corpus + corpus_size - bytes, bytes, cudaMemcpyDeviceToHost, c->stream) != cudaSuccess ||
        cudaStreamSynchronize(c->stream) != cudaSuccess)
        return ZXC_B200_ERROR_CUDA;
    return ZXC_OK;
}

extern "C" int zxg_train_literals(zxg_ctx* c, const void* const* pieces, const size_t* sizes, size_t n, const void* h_dict,
                                  uint32_t dict_size, uint32_t* h_freq, const zxg_train_src_t* src) {
    memset(h_freq, 0, 256 * sizeof(uint32_t));
    if (n == 0) return ZXC_OK;
    const u32 bs = 4096u, level = 6u; /* the reference trains at ZXC_LEVEL_DENSITY on 4 KiB slices */
    uint64_t total = 0;
    TrainSlice* h_sl = (TrainSlice*)malloc(n * sizeof(TrainSlice));
    if (!h_sl) return ZXC_ERROR_MEMORY;
    for (size_t i = 0; i < n; i++) {
        h_sl[i].off = total;
        h_sl[i].len = (u32)sizes[i];
        h_sl[i].pad = 0;
        total += sizes[i];
    }
    const size_t wstride = enc_layout(bs, (int)level).total;
    const int grid = grid_cap((n + ENC_WARPS_PER_CTA - 1) / ENC_WARPS_PER_CTA, ENC_CTAS_PER_SM);
    u8* d_src = (u8*)zxg_buffer(c, ZXG_BUF_IN, (size_t)total + 64);
    TrainSlice* d_sl = (TrainSlice*)zxg_buffer(c, ZXG_BUF_JOBS, n * sizeof(TrainSlice));
    u8* d_scratch = (u8*)zxg_buffer(c, ZXG_BUF_SCRATCH, (size_t)grid * ENC_WARPS_PER_CTA * wstride);
    u32* d_freq = (u32*)zxg_buffer(c, ZXG_BUF_AUX, 256 * sizeof(u32));
    const size_t dpad = ((size_t)dict_size + 16 + 255) & ~(size_t)255;
    const size_t dtot = dpad + (size_t)ENC_HASH_SIZE * 4 + (size_t)ENC_WINDOW * 2 + 256;
    u8* d_dict = (u8*)zxg_buffer(c, ZXG_BUF_DICT, dtot);
    if (!d_src || !d_sl || !d_scratch || !d_freq || !d_dict) {
        free(h_sl);
        return ZXC_ERROR_MEMORY;
    }
    train_events T;
    int rc = tev_init(&T, 3);
    if (rc == ZXC_OK) rc = gather_samples(c, d_src, pieces, sizes, n, src, &T);
    if (rc == ZXC_OK &&
        (cudaMemsetAsync(d_src + total, 0, 64, c->stream) != cudaSuccess ||
         cudaMemcpyAsync(d_sl, h_sl, n * sizeof(TrainSlice), cudaMemcpyHostToDevice, c->stream) != cudaSuccess ||
         cudaMemsetAsync(d_freq, 0, 256 * sizeof(u32), c->stream) != cudaSuccess ||
         cudaMemsetAsync(d_dict, 0, dtot, c->stream) != cudaSuccess ||
         cudaMemsetAsync(c->counter, 0, sizeof(unsigned long long), c->stream) != cudaSuccess))
        rc = ZXC_B200_ERROR_CUDA;
    if (rc == ZXC_OK) rc = zxg_h2d(c, d_dict, h_dict, dict_size);
    if (rc == ZXC_OK) {
        cudaEventRecord(T.ev[1], c->stream);
        EncodeParams P;
        memset(&P, 0, sizeof P);
        P.src = d_src;
        P.scratch = d_scratch;
        P.counter = c->counter;
        P.dict = d_dict;
        P.seed_head = (const u32*)(d_dict + dpad);
        P.seed_chain = (const unsigned short*)(d_dict + dpad + (size_t)ENC_HASH_SIZE * 4);
        P.scratch_stride = wstride;
        P.block_size = bs;
        P.n_blocks = (u32)n;
        P.level = level;
        P.dict_size = dict_size;
        zxc_seed_kernel<<<1, 32, 0, c->stream>>>(d_dict, dict_size, level, (u32*)P.seed_head, (unsigned short*)P.seed_chain);
        zxc_train_lit_kernel<<<grid, ENC_CTA_THREADS, 0, c->stream>>>(P, d_sl, d_freq);
        __atomic_add_fetch(&g_launches, 2, __ATOMIC_RELAXED);
        cudaEventRecord(T.ev[2], c->stream);
        if (cudaMemcpyAsync(h_freq, d_freq, 256 * sizeof(u32), cudaMemcpyDeviceToHost, c->stream) != cudaSuccess ||
            cudaStreamSynchronize(c->stream) != cudaSuccess)
            rc = ZXC_B200_ERROR_CUDA;
    }
    if (rc == ZXC_OK) {
        t_train_ms[ZXG_T_SLICES] = tev_ms(&T, 0, 1);
        t_train_ms[ZXG_T_HIST] = tev_ms(&T, 1, 2);
    } else {
        fprintf(stderr, "libzxc (CUDA build): dictionary table training failed: %s\n", cudaGetErrorString(cudaGetLastError()));
    }
    tev_free(&T);
    free(h_sl);
    return rc;
}
