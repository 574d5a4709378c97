/* af_xxcc.c -- XXCC object of the C ABI (host C; compute = kernels/bank_xxcc.cu `k_xxcc`).
 * Interface spec: src/feature/xxcc_algorithm.h:12-39, behaviour src/feature/xxcc_algorithm.c. */
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include "../af_internal.h"

struct OpaqueXXCC {
    int num, timeLength;
    float *dDctT;               /* device, transposed ortho DCT-II [num][num] */
    AfPipe pipe;
};

int xxccObj_new(XXCCObj *out, int num) {
    af_clear_error();
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
    return x->dDctT ? AF_OK : af_dct2_upload_transposed(&x->dDctT, x->num);
}

typedef struct { int num, ccNum, rectifyType, energyType, order; const float *dctT; } XxccCall;

static int xxcc_chunk(void *p, int nb, float *const *d, void *st) {
    const XxccCall *a = (const XxccCall *)p;
    return af_launch_xxcc(d[0], nb, a->num, a->ccNum, a->rectifyType, a->dctT, d[1], st);
}

int af_xxcc_batch(AfPipe *pipe, const float *in, int rows, int num, int ccNum, int rectifyType, const float *dctT,
                  float *out, int memKind, void *stream) {
    XxccCall a = {num, ccNum, rectifyType, 0, 0, dctT};
    const AfPlane pl[2] = {{in, (size_t)num, AF_IN, 0}, {out, (size_t)ccNum, AF_OUT, 0}};
    return af_run_batch(pipe, memKind, stream, xxcc_chunk, &a, pl, 2, rows, AF_PIPE_CHUNK_BYTES);
}

int xxccObj_xxccBatch(XXCCObj x, const float *in, int rows, int ccNum, int rectifyType, float *out,
                      int memKind, void *stream) {
    if (!x || !in || !out || rows < 0) return af_fail(AF_ERR_ARG, "xxccObj_xxccBatch: bad argument");
    if (ccNum < 1 || ccNum > x->num) return af_fail(AF_ERR_ARG, "xxccObj_xxccBatch: ccNum=%d outside [1, %d]", ccNum, x->num);
    af_clear_error();
    int rc = xxcc_device(x);
    if (rc) return rc;
    return af_xxcc_batch(&x->pipe, in, rows, x->num, ccNum, rectifyType, x->dDctT, out, memKind, stream);
}

void xxccObj_xxcc(XXCCObj x, float *mDataArr1, int mLength, CepstralRectifyType *rectifyType, float *mDataArr2) {
    if (!x || !mDataArr1 || !mDataArr2) return;
    if (mLength > x->num) return;                 /* silent, like xxcc_algorithm.c:116-118 */
    if (x->timeLength <= 0 || mLength < 1) return;
    xxccObj_xxccBatch(x, mDataArr1, x->timeLength, mLength, rectifyType ? (int)*rectifyType : CepstralRectify_Log,
                      mDataArr2, AFB200_MEM_HOST, NULL);
}

static int xxcc_standard_chunk(void *p, int nb, float *const *d, void *st) {
    const XxccCall *a = (const XxccCall *)p;
    return af_launch_xxcc_standard(d[0], d[1], nb, a->num, a->ccNum, a->rectifyType, a->energyType, a->order, a->dctT,
                                   d[2], d[3], d[4], st);
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
    XxccCall a = {x->num, ccNum, rectifyType, energyType, order, x->dDctT};
    const size_t W = (size_t)ccNum + (energyType == CepstralEnergy_Append ? 1 : 0);
    const AfPlane pl[5] = {{in, (size_t)x->num, AF_IN, 0}, {energy, 1, AF_IN, 0},
                           {coe, W, AF_OUT, 0}, {delta1, W, AF_OUT, 0}, {delta2, W, AF_OUT, 0}};
    return af_run_batch(&x->pipe, memKind, stream, xxcc_standard_chunk, &a, pl, 5, rows, AF_PIPE_CHUNK_BYTES);
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
    af_pipe_free(&x->pipe);
    af_dev_free(x->dDctT);
    free(x);
}
