/* af_wavelet.c -- DWTObj, WPTObj and SWTObj of the C ABI (host C; compute = kernels/wavelet.cu, one launch per level).
 * Interface specs: include/{dwt,wpt,swt}_algorithm.h, behaviour src/{dwt,wpt,swt}_algorithm.c, filters
 * src/filterbank/dwt_filterCoef.c.  The three objects share one filter lookup and one object layout; DWT and WPT keep
 * a device workspace of ping-pong level buffers, SWT reads each level's input from its own approximation rows. */
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include "../af_internal.h"
#include "../kernels/wavelet_coef_gen.h"

enum { AF_DWT = 0, AF_WPT = 1, AF_SWT = 2 };

typedef struct {
    int kind, num, log2n, n, dec;
    float lo[80], hi[80];
    float *dLo, *dHi;
    int uploaded;         /* 1 once both filters are on the device */
    AfDevBuf work;
    AfPipe pipe;
} AfWt;

struct OpaqueDWT { AfWt w; };
struct OpaqueWPT { AfWt w; };
struct OpaqueSWT { AfWt w; };

/* dwt_filterCoef.c :49-752 with the reference's (type, t1, t2) matching: Haar and DMey ignore t1 / t2, Bior reads
 * both, the others t1; a combination the reference does not list is sym4 (:734).  -2 for the listed filters this
 * library does not generate (kernels/wavelet_coef_gen.h). */
static int wt_filters(AfWt *w, const char *who, const WaveletDiscreteType *waveletType, const int *t1, const int *t2) {
    const int ty = waveletType ? (int)*waveletType : WaveletDiscrete_Sym;
    const int a = t1 ? *t1 : 4, b = t2 ? *t2 : 4;
    const int k1 = ty == WaveletDiscrete_Haar || ty == WaveletDiscrete_DMey ? 0 : a;
    const int k2 = ty == WaveletDiscrete_Bior ? b : 0;
    for (size_t i = 0; i < sizeof(af_wavelet_refusals) / sizeof(af_wavelet_refusals[0]); i++) {
        const AfWaveletRefusal *r = &af_wavelet_refusals[i];
        if (r->type == ty && r->t1 == k1 && r->t2 == k2)
            return af_fail(-2, "%s: wavelet type %d, t1=%d, t2=%d is not supported: %s", who, ty, a, b, r->why);
    }
    const AfWaveletCoef *c = NULL, *sym4 = NULL;
    for (size_t i = 0; i < sizeof(af_wavelet_coefs) / sizeof(af_wavelet_coefs[0]); i++) {
        const AfWaveletCoef *e = &af_wavelet_coefs[i];
        if (e->type == ty && e->t1 == k1 && e->t2 == k2) c = e;
        if (e->type == WaveletDiscrete_Sym && e->t1 == 4) sym4 = e;
    }
    if (!c) c = sym4;
    w->dec = c->length;
    memcpy(w->lo, c->lo, sizeof(float) * (size_t)c->length);
    memcpy(w->hi, c->hi, sizeof(float) * (size_t)c->length);
    return 0;
}

static void *wt_alloc(int kind, int num, int log2n, int n) {
    AfWt *w = (AfWt *)calloc(1, sizeof(AfWt));
    if (!w) return NULL;
    w->kind = kind; w->num = num; w->log2n = log2n; w->n = n;
    return w;
}

/* dwtObj_new / wptObj_new :55-104 */
static int wt_new_tree(void **obj, int kind, const char *who, int num, int radix2Exp, WaveletDiscreteType *waveletType,
                       int *t1, int *t2) {
    af_clear_error();
    if (!obj) return -1;
    *obj = NULL;
    if (radix2Exp && (radix2Exp < 1 || radix2Exp > 30)) return -100;
    if (num < 1 || num > radix2Exp - 1) return -1;
    if (radix2Exp > AFB200_WAVELET_MAX_EXP)
        return af_fail(-2, "%s: radix2Exp=%d; the largest supported is %d", who, radix2Exp, AFB200_WAVELET_MAX_EXP);
    AfWt f;
    int rc = wt_filters(&f, who, waveletType, t1, t2);
    if (rc) return rc;
    AfWt *w = (AfWt *)wt_alloc(kind, num, radix2Exp, 1 << radix2Exp);
    if (!w) return -1;
    w->dec = f.dec;
    memcpy(w->lo, f.lo, sizeof(f.lo));
    memcpy(w->hi, f.hi, sizeof(f.hi));
    *obj = w;
    return 0;
}

int dwtObj_new(DWTObj *dwtObj, int num, int radix2Exp, WaveletDiscreteType *waveletType, int *t1, int *t2) {
    return wt_new_tree((void **)dwtObj, AF_DWT, "dwtObj_new", num, radix2Exp, waveletType, t1, t2);
}

int wptObj_new(WPTObj *wptObj, int num, int radix2Exp, WaveletDiscreteType *waveletType, int *t1, int *t2) {
    return wt_new_tree((void **)wptObj, AF_WPT, "wptObj_new", num, radix2Exp, waveletType, t1, t2);
}

/* swt_algorithm.c :50-118 */
int swtObj_new(SWTObj *swtObj, int num, int fftLength, WaveletDiscreteType *waveletType, int *t1, int *t2) {
    af_clear_error();
    if (!swtObj) return -1;
    *swtObj = NULL;
    if (num < 0 || num > 30) return af_fail(-1, "swtObj_new: num=%d outside 0 .. 30", num);
    if (fftLength < (1 << num) || fftLength % (1 << num)) return -1;
    if (fftLength > (1 << AFB200_WAVELET_MAX_EXP))
        return af_fail(-2, "swtObj_new: fftLength=%d; the largest supported is %d", fftLength, 1 << AFB200_WAVELET_MAX_EXP);
    AfWt f;
    int rc = wt_filters(&f, "swtObj_new", waveletType, t1, t2);
    if (rc) return rc;
    AfWt *w = (AfWt *)wt_alloc(AF_SWT, num, 0, fftLength);
    if (!w) return -1;
    w->dec = f.dec;
    memcpy(w->lo, f.lo, sizeof(f.lo));
    memcpy(w->hi, f.hi, sizeof(f.hi));
    *swtObj = (SWTObj)w;
    return 0;
}

/* d[0] data nb x n, d[1] coef nb x n (SWT: approximations nb x num x n), d[2] mData (SWT: details) or NULL */
static int wt_chunk(void *ctx, int nb, float *const *d, void *st) {
    AfWt *w = (AfWt *)ctx;
    const int n = w->n, num = w->num;
    int rc;
    if (w->kind == AF_SWT) {
        const long long rs = (long long)num * n;
        for (int i = 0; i < num; i++) {
            const float *in = i ? d[1] + (long long)(i - 1) * n : d[0];
            if ((rc = af_launch_swt_level(in, i ? rs : n, w->dLo, w->dHi, w->dec, n, 1 << i, nb, d[1] + (long long)i * n,
                                          d[2] + (long long)i * n, rs, st)))
                return rc;
        }
        return AF_OK;
    }
    /* DWT: approximations alternate between the halves of an n-float buffer per clip; WPT: levels between two n-float
     * buffers.  The last level writes coef directly. */
    const long long per = w->kind == AF_WPT ? 2LL * n : n;
    if ((rc = af_devbuf_reserve(&w->work, sizeof(float) * (size_t)per * (size_t)nb))) return rc;
    float *ws = (float *)w->work.ptr;
    const long long half = w->kind == AF_WPT ? n : n / 2;
    for (int i = 0; i < num; i++) {
        AfWaveletLevel a;
        a.L = n >> i;
        a.in = i ? ws + ((i - 1) % 2 ? half : 0) : d[0];
        a.inStride = i ? per : n;
        float *next = i == num - 1 ? d[1] : ws + (i % 2 ? half : 0);
        a.lo = next;
        a.loStride = i == num - 1 ? n : per;
        if (w->kind == AF_WPT) {
            a.nodes = 1 << i; a.nodeBase = (1 << i) - 1; a.wpt = 1;
            a.hi = next; a.hiStride = a.loStride;
        } else {
            a.nodes = 1; a.nodeBase = 0; a.wpt = 0;
            a.hi = d[1]; a.hiStride = n;
        }
        a.loD = w->dLo; a.hiD = w->dHi; a.dec = w->dec; a.batch = nb;
        if ((rc = af_launch_wavelet_level(&a, st))) return rc;
    }
    if (d[2]) return af_launch_wavelet_expand(d[1], w->log2n, w->kind == AF_WPT ? 1 << num : num, w->kind == AF_WPT,
                                              nb, d[2], st);
    return AF_OK;
}

static int wt_batch(AfWt *w, const char *who, const float *data, int batch, float *out1, float *out2, int memKind,
                    void *stream) {
    if (!w || !data || !out1 || (w->kind == AF_SWT && !out2) || batch < 0)
        return af_fail(AF_ERR_ARG, "%s: bad argument", who);
    af_clear_error();
    int rc = af_device_ready();
    if (rc) return rc;
    if (!w->uploaded) {          /* both again after a failure: af_dev_upload frees what an earlier attempt left */
        if ((rc = af_dev_upload((void **)&w->dLo, w->lo, sizeof(float) * (size_t)w->dec)) ||
            (rc = af_dev_upload((void **)&w->dHi, w->hi, sizeof(float) * (size_t)w->dec)))
            return rc;
        w->uploaded = 1;
    }
    if (batch == 0 || (w->kind == AF_SWT && w->num == 0)) return AF_OK;
    const size_t rows = w->kind == AF_SWT ? (size_t)w->num : w->kind == AF_WPT ? (size_t)1 << w->num : (size_t)w->num;
    const size_t n = (size_t)w->n;
    const AfPlane pl[3] = {{data, n, AF_IN, 0},
                           {out1, w->kind == AF_SWT ? rows * n : n, AF_OUT, 0},
                           {out2, rows * n, AF_OUT, 0}};
    return af_run_batch(&w->pipe, memKind, stream, wt_chunk, w, pl, 3, batch, AF_PIPE_CHUNK_BYTES);
}

int dwtObj_dwtBatch(DWTObj o, const float *data, int batch, float *coef, float *mData, int memKind, void *stream) {
    return wt_batch(o ? &o->w : NULL, "dwtObj_dwtBatch", data, batch, coef, mData, memKind, stream);
}

int wptObj_wptBatch(WPTObj o, const float *data, int batch, float *coef, float *mData, int memKind, void *stream) {
    return wt_batch(o ? &o->w : NULL, "wptObj_wptBatch", data, batch, coef, mData, memKind, stream);
}

int swtObj_swtBatch(SWTObj o, const float *data, int batch, float *mData1, float *mData2, int memKind, void *stream) {
    return wt_batch(o ? &o->w : NULL, "swtObj_swtBatch", data, batch, mData1, mData2, memKind, stream);
}

void dwtObj_dwt(DWTObj o, float *dataArr, float *coefArr, float *mDataArr) {
    dwtObj_dwtBatch(o, dataArr, 1, coefArr, mDataArr, AFB200_MEM_HOST, NULL);
}

void wptObj_wpt(WPTObj o, float *dataArr, float *coefArr, float *mDataArr) {
    wptObj_wptBatch(o, dataArr, 1, coefArr, mDataArr, AFB200_MEM_HOST, NULL);
}

void swtObj_swt(SWTObj o, float *dataArr, float *mDataArr1, float *mDataArr2) {
    swtObj_swtBatch(o, dataArr, 1, mDataArr1, mDataArr2, AFB200_MEM_HOST, NULL);
}

static void wt_free(AfWt *w) {
    if (!w) return;
    af_pipe_free(&w->pipe);
    af_devbuf_free(&w->work);
    af_dev_free(w->dLo);
    af_dev_free(w->dHi);
    free(w);
}

void dwtObj_free(DWTObj o) { wt_free(o ? &o->w : NULL); }
void wptObj_free(WPTObj o) { wt_free(o ? &o->w : NULL); }
void swtObj_free(SWTObj o) { wt_free(o ? &o->w : NULL); }
