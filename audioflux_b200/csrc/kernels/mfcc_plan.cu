// mfcc_plan.cu -- host side of the fused MFCC: which kernel serves a call, and the one plan type over the two kernels'
// own plans (mfcc_fused.cu = v1, mfcc_fused2.cu = v2).
#include <string.h>
#include "mfcc_common.cuh"

struct AfMfccPlan {
    int kernel;         // AF_MFCC_V1 | AF_MFCC_V2
    int bankOnly;       // 1: the kernel stops after the filter bank
    void *impl;         // the kernel file's plan
};

int af_mfcc_route(const AfMfccCall *c) {
    if (c->bankOnly && (!c->realMode || getenv("AFB200_BFT_GENERAL")))     // complex mode / test hook: composed path
        return AF_MFCC_COMPOSED;
    if (c->reassign || c->normValue != 1.0f || c->linear || !c->banded || c->slideLength % 4 || c->dataLength % 4 ||
        (reinterpret_cast<uintptr_t>(c->data) & 15))                      // (TMA bulk copies of the clips)
        return AF_MFCC_COMPOSED;
    // fftLength 2048, num <= 128, ccNum 1 .. 64 and a bank v1's weight table holds
    if (!af_mfcc1_supported(c->fftLength, c->num, c->bankOnly ? 1 : c->ccNum, c->bands)) return AF_MFCC_COMPOSED;
    // v2 is only ever tried on banks v1's planner accepts.  Banks v1 rejects (Bark / Slaney / BandWidth-128) may or may
    // not have v2's two-overlap structure; they keep the composed path until that is checked and measured.
    const char *k = getenv("AFB200_MFCC_KERNEL");                          // test hook: "v1" keeps v2 out
    if (k && !strcmp(k, "v1")) return AF_MFCC_V1;
    if (!*c->v2Bank) *c->v2Bank = af_mfcc2_supported(c->fftLength, c->num, 1, c->bank) ? 1 : -1;
    return *c->v2Bank > 0 ? AF_MFCC_V2 : AF_MFCC_V1;
}

int af_mfcc_plan_build(AfMfccPlan **plan, int kernel, int bankOnly, int fftLength, int num, int ccNum,
                       const float *window, const float *bank, const AfBands *bands, int dataType) {
    *plan = NULL;
    AfMfccPlan *pl = static_cast<AfMfccPlan *>(calloc(1, sizeof(AfMfccPlan)));
    const int cc = bankOnly ? 1 : ccNum;                 // a bank-only plan carries a zero DCT row its kernel never reads
    float *dct = static_cast<float *>(calloc((size_t)cc * num, sizeof(float)));
    if (!pl || !dct) { free(pl); free(dct); return AF_ERR_NOMEM; }
    if (!bankOnly) af_dct2_matrix(num, cc, dct);
    pl->kernel = kernel; pl->bankOnly = bankOnly;
    const int rc = kernel == AF_MFCC_V2 ? af_mfcc2_plan_build(&pl->impl, fftLength, num, cc, window, bank, dct, dataType)
                                        : af_mfcc1_plan_build(&pl->impl, fftLength, num, cc, window, bank, bands, dct, dataType);
    free(dct);
    if (rc) { free(pl); return rc; }
    *plan = pl;
    return AF_OK;
}

int af_mfcc_plan_kind(const AfMfccPlan *plan) { return plan ? plan->kernel : AF_MFCC_COMPOSED; }

void af_mfcc_plan_free(AfMfccPlan *plan) {
    if (!plan) return;
    if (plan->kernel == AF_MFCC_V2) af_mfcc2_plan_free(plan->impl);
    else af_mfcc1_plan_free(plan->impl);
    free(plan);
}

int af_launch_mfcc(const AfMfccPlan *plan, const float *data, int dataLength, int batch, int timeLength, int slideLength,
                   int rectifyType, float *out, int nPeer, float *const *peerOut, void *stream) {
    if (!plan) return af_fail(AF_ERR_ARG, "fused MFCC: no plan");
    if (batch <= 0 || timeLength <= 0) return AF_OK;
    if (slideLength % 4 || dataLength % 4 || (reinterpret_cast<uintptr_t>(data) & 15))
        return af_fail(AF_ERR_UNSUPPORTED, "fused MFCC needs 16-byte aligned clips and slideLength %% 4 == 0 (TMA bulk copy)");
    if (nPeer < 0 || nPeer > kMfccMaxPeers || (nPeer > 0 && !peerOut))
        return af_fail(AF_ERR_ARG, "fused MFCC: nPeer=%d outside [0, %d]", nPeer, kMfccMaxPeers);
    return (plan->kernel == AF_MFCC_V2 ? af_mfcc2_launch : af_mfcc1_launch)(
        plan->impl, data, dataLength, batch, timeLength, slideLength, rectifyType, out, nPeer, peerOut, plan->bankOnly, stream);
}
