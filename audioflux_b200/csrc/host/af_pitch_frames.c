/* af_pitch_frames.c -- the core the frame-wise pitch trackers share (af_pitch_pef.c, af_pitch_yin.c,
 * af_pitch_ncf_cep.c): the constructor's parameter rules, the frame count with the streaming carry, the batched call's
 * entry and the legacy call's input.  Behaviour: src/mir/_pitch_{pef,yin,ncf,cep}.c's new and pitch functions
 * (restated in include/afb200_pitch_*.h). */
#include "../af_internal.h"

int af_pitch_frames_init(AfPitchFrames *f, float *lf, float *hf, const AfPitchRules *r, const int *samplate,
                         const float *lowFre, const float *highFre, const int *radix2Exp, const int *slideLength,
                         const int *isContinue) {
    const int sr = samplate && *samplate > 0 && *samplate <= 196000 ? *samplate : 32000;
    *lf = lowFre && *lowFre >= 27 ? *lowFre : r->lowFre;
    *hf = r->highFre;
    if (highFre) {
        if (*highFre > *lf && *highFre < sr / 2) *hf = *highFre;
        else { *lf = r->lowFre; *hf = r->highReset; }
    }
    const int log2n = radix2Exp && *radix2Exp >= 1 && *radix2Exp <= 30 ? *radix2Exp : 12;
    if (log2n > r->maxExp) {
        af_fail(-2, "%s: radix2Exp=%d; the largest supported is %d (%s)", r->who, log2n, r->maxExp, r->why);
        return -2;
    }
    const int n = 1 << log2n;
    int slide = slideLength && *slideLength > 0 ? *slideLength : n / 4;
    if (slide < 1) slide = 1;                                   /* n/4 at n = 2: the reference divides by zero */
    *f = (AfPitchFrames){sr, log2n, n, slide, isContinue ? *isContinue : 0, {0}, {0}};
    return 0;
}

int af_pitch_frames(const AfPitchFrames *f, int dataLength) {
    return dataLength < f->n ? 0 : (dataLength - f->n) / f->slideLength + 1;
}

int af_pitch_time_length(const AfPitchFrames *f, int dataLength) {
    if (!f) return 0;
    return af_pitch_frames(f, f->isContinue ? dataLength + f->tail.length : dataLength);
}

int af_pitch_batch_begin(const AfPitchFrames *f, const char *who, const float *data, int dataLength, int batch,
                         const float *fre, int *T) {
    *T = f && dataLength > 0 ? af_pitch_frames(f, dataLength) : 0;
    if (!f || !data || (!fre && *T > 0 && batch > 0) || dataLength <= 0 || batch < 0)   /* fre may be NULL when empty */
        return af_fail(AF_ERR_ARG, "%s: bad argument", who);
    af_clear_error();
    if (batch == 0) *T = 0;
    return af_device_ready();
}

int af_pitch_legacy_input(AfPitchFrames *f, const float *data, int dataLength, const float **x, int *len) {
    if (!f) return 0;
    af_clear_error();
    if (!data || dataLength <= 0) return 0;
    *x = data;
    *len = dataLength;
    if (f->isContinue && !af_tail_assemble(&f->tail, f->n, f->slideLength, data, dataLength, x, len)) return 0;
    return af_pitch_frames(f, *len);
}

void af_pitch_frames_free(AfPitchFrames *f) {
    af_pipe_free(&f->pipe);
    af_tail_free(&f->tail);
}
