/* af_ctx.c -- device context, error reporting and device-memory helpers (host C over the CUDA
 * runtime API).  There is no CPU compute path in this library: every compute entry point ends
 * in a kernel launch or fails with a recorded message. */
#include <stdarg.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <cuda_runtime_api.h>
#include "../af_internal.h"

#define AFB200_VERSION 100   /* 0.1.0 */

static __thread char g_err[512];
static __thread int g_device = -1;          /* -1: follow the CUDA current device */
static long long g_launches = 0;

int af_fail(int code, const char *fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
    fprintf(stderr, "[audioflux_b200] error %d: %s\n", code, g_err);
    return code;
}

void af_clear_error(void) { g_err[0] = 0; }
const char *afb200_lastError(void) { return g_err; }
int afb200_version(void) { return AFB200_VERSION; }

int af_cuda_check(int e, const char *what) {
    if (e == cudaSuccess) return AF_OK;
    return af_fail(AF_ERR_CUDA, "%s: %s", what, cudaGetErrorString((cudaError_t)e));
}

int afb200_deviceCount(void) {
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess) { cudaGetLastError(); return 0; }
    return n;
}

int afb200_setDevice(int device) {
    int n = afb200_deviceCount();
    if (device < 0 || device >= n) return af_fail(AF_ERR_ARG, "afb200_setDevice(%d): %d device(s) visible", device, n);
    g_device = device;
    return af_cuda_check(cudaSetDevice(device), "cudaSetDevice");
}

int afb200_getDevice(void) {
    int d = -1;
    if (cudaGetDevice(&d) != cudaSuccess) { cudaGetLastError(); return -1; }
    return d;
}

int af_device_ready(void) {
    if (afb200_deviceCount() <= 0)
        return af_fail(AF_ERR_NOGPU, "no CUDA device is visible: libaudioflux_b200 has no CPU fallback");
    if (g_device >= 0) return af_cuda_check(cudaSetDevice(g_device), "cudaSetDevice");
    return AF_OK;
}

int afb200_deviceSynchronize(void) { return af_cuda_check(cudaDeviceSynchronize(), "cudaDeviceSynchronize"); }
long long afb200_kernelLaunchCount(void) { return g_launches; }
void af_count_launch(int n) { __sync_fetch_and_add(&g_launches, (long long)n); }

int af_devbuf_reserve(AfDevBuf *b, size_t bytes) {
    if (b->bytes >= bytes && b->ptr) return AF_OK;
    if (b->ptr) { cudaFree(b->ptr); b->ptr = NULL; b->bytes = 0; }
    if (bytes == 0) return AF_OK;
    int e = cudaMalloc(&b->ptr, bytes);
    if (e != cudaSuccess) { b->ptr = NULL; return af_fail(AF_ERR_NOMEM, "cudaMalloc(%zu bytes): %s", bytes, cudaGetErrorString((cudaError_t)e)); }
    b->bytes = bytes;
    return AF_OK;
}

void af_devbuf_free(AfDevBuf *b) { if (b->ptr) cudaFree(b->ptr); b->ptr = NULL; b->bytes = 0; }

/* *dptr must be NULL or an earlier allocation of this call (object fields: calloc'ed); a table uploaded again after a
 * failed lazy initialisation replaces the earlier copy instead of leaking it (ADVICE r1) */
int af_dev_upload(void **dptr, const void *host, size_t bytes) {
    if (*dptr) { cudaFree(*dptr); }
    *dptr = NULL;
    if (bytes == 0) return AF_OK;
    int e = cudaMalloc(dptr, bytes);
    if (e != cudaSuccess) { *dptr = NULL; return af_fail(AF_ERR_NOMEM, "cudaMalloc(%zu bytes): %s", bytes, cudaGetErrorString((cudaError_t)e)); }
    e = cudaMemcpy(*dptr, host, bytes, cudaMemcpyHostToDevice);
    /* A pageable-source cudaMemcpy may return once the bytes sit in the driver's staging buffer, before the DMA has
     * landed; the kernels that read the table run on non-blocking streams, which do not order themselves behind the
     * legacy stream.  Wait for the copy itself (tables are uploaded once per object, never on a hot path). */
    if (e == cudaSuccess) e = cudaStreamSynchronize(cudaStreamLegacy);
    return af_cuda_check(e, "cudaMemcpy H2D (table)");
}

void af_dev_free(void *p) { if (p) cudaFree(p); }

static int af_stream_create(void **s) {
    if (*s) return AF_OK;                                  /* already created by an earlier, partially failed initialisation */
    cudaStream_t st;
    int e = cudaStreamCreateWithFlags(&st, cudaStreamNonBlocking);
    if (e != cudaSuccess) { *s = NULL; return af_cuda_check(e, "cudaStreamCreate"); }
    *s = (void *)st;
    return AF_OK;
}
static void af_stream_destroy(void *s) { if (s) cudaStreamDestroy((cudaStream_t)s); }
int af_stream_sync(void *s) { return af_cuda_check(cudaStreamSynchronize((cudaStream_t)s), "cudaStreamSynchronize"); }
int af_memcpy_h2d(void *d, const void *h, size_t n, void *s) {
    return af_cuda_check(cudaMemcpyAsync(d, h, n, cudaMemcpyHostToDevice, (cudaStream_t)s), "cudaMemcpyAsync H2D");
}
int af_memset_d(void *d, int v, size_t n, void *s) {
    return af_cuda_check(cudaMemsetAsync(d, v, n, (cudaStream_t)s), "cudaMemsetAsync");
}
size_t af_dev_free_bytes(void) {
    size_t f = 0, t = 0;
    if (cudaMemGetInfo(&f, &t) != cudaSuccess) { cudaGetLastError(); return 0; }
    return f;
}
int af_sm_count(void) {
    int d = 0, n = 0;
    if (cudaGetDevice(&d) != cudaSuccess) return 0;
    if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, d) != cudaSuccess) return 0;
    return n;
}

/* ---- events: ordering between the copy / compute / read-back streams of the host-pointer pipelines ---- */
static int af_event_create(void **ev) {
    cudaEvent_t e;
    int rc = cudaEventCreateWithFlags(&e, cudaEventDisableTiming);
    if (rc != cudaSuccess) { *ev = NULL; return af_cuda_check(rc, "cudaEventCreate"); }
    *ev = (void *)e;
    return AF_OK;
}
static void af_event_destroy(void *ev) { if (ev) cudaEventDestroy((cudaEvent_t)ev); }
static int af_event_record(void *ev, void *stream) { return af_cuda_check(cudaEventRecord((cudaEvent_t)ev, (cudaStream_t)stream), "cudaEventRecord"); }
static int af_stream_wait_event(void *stream, void *ev) { return af_cuda_check(cudaStreamWaitEvent((cudaStream_t)stream, (cudaEvent_t)ev, 0), "cudaStreamWaitEvent"); }

static size_t plane_floats(const AfPlane *p) { return p->per * (size_t)(p->layers > 1 ? p->layers : 1); }

/* items c0 .. c0+nb-1 of a plane between caller memory and a slot (device layout layers x nb x per) */
static int plane_copy(const AfPlane *p, float *dev, int c0, int nb, int batch, int toDevice, void *st) {
    const size_t w = sizeof(float) * p->per * nb, hostPitch = sizeof(float) * p->per * batch;
    char *host = (char *)p->ptr + sizeof(float) * p->per * c0;
    int e;
    if (p->layers > 1)
        e = toDevice ? cudaMemcpy2DAsync(dev, w, host, hostPitch, w, p->layers, cudaMemcpyHostToDevice, (cudaStream_t)st)
                     : cudaMemcpy2DAsync(host, hostPitch, dev, w, w, p->layers, cudaMemcpyDeviceToHost, (cudaStream_t)st);
    else
        e = toDevice ? cudaMemcpyAsync(dev, host, w, cudaMemcpyHostToDevice, (cudaStream_t)st)
                     : cudaMemcpyAsync(host, dev, w, cudaMemcpyDeviceToHost, (cudaStream_t)st);
    return af_cuda_check(e, toDevice ? "cudaMemcpyAsync H2D" : "cudaMemcpyAsync D2H");
}

static int pipe_chunks(AfPipe *pp, AfChunkFn fn, void *ctx, const AfPlane *pl, int np, int batch, int chunk, void *st) {
    int rc, inout = 0;
    for (int i = 0; i < np; i++) inout |= pl[i].ptr && pl[i].dir == AF_INOUT;
    for (int s = 0; s < (chunk < batch ? 2 : 1); s++)              /* the second slot only when a second chunk exists */
        for (int i = 0; i < np; i++)
            if (pl[i].ptr && (rc = af_devbuf_reserve(&pp->slot[s][i], sizeof(float) * plane_floats(&pl[i]) * chunk))) return rc;
    int k = 0;
    for (int c0 = 0; c0 < batch; c0 += chunk, k++) {
        const int nb = batch - c0 < chunk ? batch - c0 : chunk, s = k & 1;
        float *d[AF_PIPE_MAX_PLANES];
        for (int i = 0; i < np; i++) d[i] = pl[i].ptr ? (float *)pp->slot[s][i].ptr : NULL;
        if (k >= 2) {                                   /* slot reuse: its previous transform and read-back are over */
            if ((rc = af_stream_wait_event(pp->inStream, pp->evDone[s])) || (rc = af_stream_wait_event(st, pp->evOut[s]))) return rc;
            if (inout && (rc = af_stream_wait_event(pp->inStream, pp->evOut[s]))) return rc;
        }
        for (int i = 0; i < np; i++)
            if (pl[i].ptr && (pl[i].dir & AF_IN) && (rc = plane_copy(&pl[i], d[i], c0, nb, batch, 1, pp->inStream))) return rc;
        if ((rc = af_event_record(pp->evIn[s], pp->inStream)) || (rc = af_stream_wait_event(st, pp->evIn[s]))) return rc;
        if ((rc = fn(ctx, nb, d, st))) return rc;
        if ((rc = af_event_record(pp->evDone[s], st)) || (rc = af_stream_wait_event(pp->outStream, pp->evDone[s]))) return rc;
        for (int i = 0; i < np; i++)
            if (pl[i].ptr && (pl[i].dir & AF_OUT) && (rc = plane_copy(&pl[i], d[i], c0, nb, batch, 0, pp->outStream))) return rc;
        if ((rc = af_event_record(pp->evOut[s], pp->outStream))) return rc;
    }
    return AF_OK;
}

int af_run_batch(AfPipe *pp, int memKind, void *stream, AfChunkFn fn, void *ctx, const AfPlane *pl, int np, int batch,
                 size_t chunkBytes) {
    if (np > AF_PIPE_MAX_PLANES) return af_fail(AF_ERR_ARG, "af_run_batch: %d planes", np);
    if (memKind == AFB200_MEM_DEVICE) {                /* asynchronous on the caller's stream (NULL = the default stream) */
        float *d[AF_PIPE_MAX_PLANES];
        for (int i = 0; i < np; i++) d[i] = (float *)pl[i].ptr;
        return fn(ctx, batch, d, stream);
    }
    int rc;
    if (!pp->ready) {
        if ((rc = af_stream_create(&pp->stream)) || (rc = af_stream_create(&pp->inStream)) || (rc = af_stream_create(&pp->outStream))) return rc;
        for (int s = 0; s < 2; s++)
            if ((rc = af_event_create(&pp->evIn[s])) || (rc = af_event_create(&pp->evDone[s])) || (rc = af_event_create(&pp->evOut[s]))) return rc;
        pp->ready = 1;
    }
    size_t inB = 0, outB = 0;
    for (int i = 0; i < np; i++) {
        if (!pl[i].ptr) continue;
        if (pl[i].dir & AF_IN) inB += sizeof(float) * plane_floats(&pl[i]);
        if (pl[i].dir & AF_OUT) outB += sizeof(float) * plane_floats(&pl[i]);
    }
    const size_t big = inB > outB ? inB : outB;
    long long per = (long long)(chunkBytes / (big > 0 ? big : 1));
    if (per >= 16) per -= per % 16;
    if (per < 1) per = 1;
    if (per > batch) per = batch;
    void *st = stream ? stream : pp->stream;
    rc = batch > 0 ? pipe_chunks(pp, fn, ctx, pl, np, batch, (int)per, st) : AF_OK;
    /* wait for all three streams whatever happened: no copy touches caller memory after the call returns */
    const int e1 = cudaStreamSynchronize((cudaStream_t)pp->inStream), e2 = cudaStreamSynchronize((cudaStream_t)st),
              e3 = cudaStreamSynchronize((cudaStream_t)pp->outStream);
    if (rc) return rc;
    return af_cuda_check(e1 ? e1 : e2 ? e2 : e3, "cudaStreamSynchronize");
}

int af_chunk_clips(size_t perClip, size_t cap, int batch) {
    size_t budget = af_dev_free_bytes() / 4;
    if (budget < perClip) budget = perClip;
    if (budget > cap) budget = cap;
    int chunk = (int)(budget / perClip);
    if (chunk < 1) chunk = 1;
    return chunk > batch ? batch : chunk;
}

int af_fence_record(void **ev, void *stream) {
    int rc;
    if (!*ev && (rc = af_event_create(ev))) return rc;
    return af_event_record(*ev, stream);
}
int af_fence_order(void *ev, void *stream) { return ev ? af_stream_wait_event(stream, ev) : AF_OK; }
int af_fence_wait(void *ev) { return ev ? af_cuda_check(cudaEventSynchronize((cudaEvent_t)ev), "cudaEventSynchronize") : AF_OK; }
void af_fence_free(void *ev) { af_event_destroy(ev); }

void af_pipe_free(AfPipe *pp) {
    af_stream_destroy(pp->stream); af_stream_destroy(pp->inStream); af_stream_destroy(pp->outStream);
    for (int s = 0; s < 2; s++) {
        af_event_destroy(pp->evIn[s]); af_event_destroy(pp->evDone[s]); af_event_destroy(pp->evOut[s]);
        for (int i = 0; i < AF_PIPE_MAX_PLANES; i++) af_devbuf_free(&pp->slot[s][i]);
    }
    memset(pp, 0, sizeof(*pp));
}

/* ---- buffers that other processes (one per GPU) can map: the gathered result of the multi-GPU path ---- */
int afb200_peerAlloc(void **devPtr, size_t bytes) {
    if (!devPtr || bytes == 0) return af_fail(AF_ERR_ARG, "afb200_peerAlloc: bad argument");
    int rc = af_device_ready();
    if (rc) return rc;
    *devPtr = NULL;
    int e = cudaMalloc(devPtr, bytes);          /* plain cudaMalloc: exportable with cudaIpcGetMemHandle at offset 0 */
    if (e != cudaSuccess) { *devPtr = NULL; return af_fail(AF_ERR_NOMEM, "cudaMalloc(%zu bytes): %s", bytes, cudaGetErrorString((cudaError_t)e)); }
    return AF_OK;
}
int afb200_peerFree(void *devPtr) { return devPtr ? af_cuda_check(cudaFree(devPtr), "cudaFree") : AF_OK; }
int afb200_ipcGetHandle(void *devPtr, void *handle64) {
    if (!devPtr || !handle64) return af_fail(AF_ERR_ARG, "afb200_ipcGetHandle: bad argument");
    cudaIpcMemHandle_t h;
    int e = cudaIpcGetMemHandle(&h, devPtr);
    if (e != cudaSuccess) return af_cuda_check(e, "cudaIpcGetMemHandle");
    memcpy(handle64, &h, sizeof(h));
    return AF_OK;
}
int afb200_ipcOpenHandle(const void *handle64, void **devPtr) {
    if (!handle64 || !devPtr) return af_fail(AF_ERR_ARG, "afb200_ipcOpenHandle: bad argument");
    int rc = af_device_ready();
    if (rc) return rc;
    cudaIpcMemHandle_t h;
    memcpy(&h, handle64, sizeof(h));
    *devPtr = NULL;
    return af_cuda_check(cudaIpcOpenMemHandle(devPtr, h, cudaIpcMemLazyEnablePeerAccess), "cudaIpcOpenMemHandle");
}
int afb200_ipcCloseHandle(void *devPtr) { return devPtr ? af_cuda_check(cudaIpcCloseMemHandle(devPtr), "cudaIpcCloseMemHandle") : AF_OK; }
