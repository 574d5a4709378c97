/* af_xxcc.c -- XXCC object of the C ABI (host C; compute = kernels/bank_xxcc.cu `k_xxcc`).
 * Interface spec: src/feature/xxcc_algorithm.h:12-39, behaviour src/feature/xxcc_algorithm.c. */
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include "../af_internal.h"

struct OpaqueXXCC {
    int num, timeLength;
    int devReady;
    void *stream;
    float *dDctT;               /* device, transposed ortho DCT-II [num][num] */
    AfDevBuf dIn, dOut, dEnergy, dD1, dD2;
};

int xxccObj_new(XXCCObj *out, int num) {
    if (!out) return -1;
    *out = NULL;
    if (num < 2) { printf("num is error!!!\n"); return -1; }
    XXCCObj x = (XXCCObj)calloc(1, sizeof(struct OpaqueXXCC));
    if (!x) return -1;
    x->num = num;
    *out = x;
    return 0;
}

void xxccObj_setTimeLength(XXCCObj x, int timeLength) { if (x) x->timeLength = timeLength; }

static int xxcc_device(XXCCObj x) {
    int rc = af_device_ready();
    if (rc) return rc;
    if (x->devReady) return AF_OK;
    if ((rc = af_stream_create(&x->stream))) return rc;
    const int n = x->num;
    float *d = (float *)malloc(sizeof(float) * (size_t)n * n), *t = (float *)malloc(sizeof(float) * (size_t)n * n);
    if (!d || !t) { free(d); free(t); return AF_ERR_NOMEM; }
    af_dct2_matrix(n, n, d);
    for (int k = 0; k < n; k++) for (int j = 0; j < n; j++) t[(size_t)j * n + k] = d[(size_t)k * n + j];
    rc = af_dev_upload((void **)&x->dDctT, t, sizeof(float) * (size_t)n * n);
    free(d); free(t);
    if (rc) return rc;
    x->devReady = 1;
    return AF_OK;
}

int xxccObj_xxccBatch(XXCCObj x, const float *in, int rows, int ccNum, int rectifyType, float *out,
                      int memKind, void *stream) {
    if (!x || !in || !out || rows < 0) return af_fail(AF_ERR_ARG, "xxccObj_xxccBatch: bad argument");
    if (ccNum < 1 || ccNum > x->num) return af_fail(AF_ERR_ARG, "xxccObj_xxccBatch: ccNum=%d outside [1, %d]", ccNum, x->num);
    af_clear_error();
    int rc = xxcc_device(x);
    if (rc) return rc;
    void *st = stream ? stream : x->stream;
    if (memKind == AFB200_MEM_DEVICE) {
        st = stream;                      /* NULL = the CUDA default stream */
        if ((rc = af_launch_xxcc(in, rows, x->num, ccNum, rectifyType, x->dDctT, out, st))) return rc;
        return AF_OK;                       /* asynchronous on the caller's stream */
    }
    size_t inB = sizeof(float) * (size_t)rows * x->num, outB = sizeof(float) * (size_t)rows * ccNum;
    if ((rc = af_devbuf_reserve(&x->dIn, inB)) || (rc = af_devbuf_reserve(&x->dOut, outB))) return rc;
    if ((rc = af_memcpy_h2d(x->dIn.ptr, in, inB, st))) return rc;
    if ((rc = af_launch_xxcc((const float *)x->dIn.ptr, rows, x->num, ccNum, rectifyType, x->dDctT, (float *)x->dOut.ptr, st))) return rc;
    if ((rc = af_memcpy_d2h(out, x->dOut.ptr, outB, st))) return rc;
    return af_stream_sync(st);
}

void xxccObj_xxcc(XXCCObj x, float *mDataArr1, int mLength, CepstralRectifyType *rectifyType, float *mDataArr2) {
    if (!x || !mDataArr1 || !mDataArr2) return;
    if (mLength > x->num) return;                 /* silent, like xxcc_algorithm.c:116-118 */
    if (x->timeLength <= 0 || mLength < 1) return;
    xxccObj_xxccBatch(x, mDataArr1, x->timeLength, mLength, rectifyType ? (int)*rectifyType : CepstralRectify_Log,
                      mDataArr2, AFB200_MEM_HOST, NULL);
}

/* batched form of xxccObj_xxccStandard (xxcc_algorithm.c:168-296).  in: rows x num, energy: rows (may be NULL
 * when energyType = Ignore); coe / delta1 / delta2: rows x (ccNum, or ccNum+1 when energyType = Append). */
int xxccObj_xxccStandardBatch(XXCCObj x, const float *in, const float *energy, int rows, int ccNum,
                              int deltaWindowLength, int energyType, int rectifyType,
                              float *coe, float *delta1, float *delta2, int memKind, void *stream) {
    if (!x || !in || !coe || !delta1 || !delta2 || rows < 0) return af_fail(AF_ERR_ARG, "xxccObj_xxccStandardBatch: bad argument");
    if (ccNum < 1 || ccNum > x->num) return af_fail(AF_ERR_ARG, "xxccObj_xxccStandardBatch: ccNum=%d outside [1, %d]", ccNum, x->num);
    if (energyType < CepstralEnergy_Replace || energyType > CepstralEnergy_Ignore)
        return af_fail(AF_ERR_ARG, "xxccObj_xxccStandardBatch: energyType=%d", energyType);
    if (energyType != CepstralEnergy_Ignore && !energy) return af_fail(AF_ERR_ARG, "xxccObj_xxccStandardBatch: energy array required");
    int order = 9;                                         /* :170, :205-209 */
    if (deltaWindowLength >= 3 && deltaWindowLength % 2 == 1) order = deltaWindowLength;
    af_clear_error();
    int rc = xxcc_device(x);
    if (rc) return rc;
    void *st = stream ? stream : x->stream;
    const int W = ccNum + (energyType == CepstralEnergy_Append ? 1 : 0);
    if (memKind == AFB200_MEM_DEVICE)
        return af_launch_xxcc_standard(in, energy, rows, x->num, ccNum, rectifyType, energyType, order, x->dDctT,
                                       coe, delta1, delta2, stream);
    const size_t inB = sizeof(float) * (size_t)rows * x->num, outB = sizeof(float) * (size_t)rows * W;
    if ((rc = af_devbuf_reserve(&x->dIn, inB)) || (rc = af_devbuf_reserve(&x->dOut, outB)) ||
        (rc = af_devbuf_reserve(&x->dD1, outB)) || (rc = af_devbuf_reserve(&x->dD2, outB)) ||
        (rc = af_devbuf_reserve(&x->dEnergy, sizeof(float) * (size_t)(rows > 0 ? rows : 1)))) return rc;
    if ((rc = af_memcpy_h2d(x->dIn.ptr, in, inB, st))) return rc;
    if (energy && (rc = af_memcpy_h2d(x->dEnergy.ptr, energy, sizeof(float) * (size_t)rows, st))) return rc;
    if ((rc = af_launch_xxcc_standard((const float *)x->dIn.ptr, (const float *)x->dEnergy.ptr, rows, x->num, ccNum,
                                      rectifyType, energyType, order, x->dDctT, (float *)x->dOut.ptr,
                                      (float *)x->dD1.ptr, (float *)x->dD2.ptr, st))) return rc;
    if ((rc = af_memcpy_d2h(coe, x->dOut.ptr, outB, st)) || (rc = af_memcpy_d2h(delta1, x->dD1.ptr, outB, st)) ||
        (rc = af_memcpy_d2h(delta2, x->dD2.ptr, outB, st))) return rc;
    return af_stream_sync(st);
}

void xxccObj_xxccStandard(XXCCObj x, float *mDataArr1, int mLength, float *energyArr, int *deltaWindowLength,
                          CepstralEnergyType *energyType, CepstralRectifyType *rectifyType,
                          float *mCoeArr, float *mDeltaArr1, float *mDeltaArr2) {
    if (!x || !mDataArr1 || !mCoeArr || !mDeltaArr1 || !mDeltaArr2) return;
    if (mLength > x->num) return;                 /* silent, like xxcc_algorithm.c:196-198 */
    if (x->timeLength <= 0 || mLength < 1) return;
    xxccObj_xxccStandardBatch(x, mDataArr1, energyArr, x->timeLength, mLength,
                              deltaWindowLength ? *deltaWindowLength : 9,
                              energyType ? (int)*energyType : CepstralEnergy_Replace,
                              rectifyType ? (int)*rectifyType : CepstralRectify_Log,
                              mCoeArr, mDeltaArr1, mDeltaArr2, AFB200_MEM_HOST, NULL);
}

void xxccObj_free(XXCCObj x) {
    if (!x) return;
    af_devbuf_free(&x->dIn); af_devbuf_free(&x->dOut);
    af_devbuf_free(&x->dEnergy); af_devbuf_free(&x->dD1); af_devbuf_free(&x->dD2);
    af_dev_free(x->dDctT);
    af_stream_destroy(x->stream);
    free(x);
}
