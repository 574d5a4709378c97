/* afb200_types.h -- enum ints of the audioFlux C ABI used by the time-frequency hot path.
 *
 * Replaces: src/flux_base.h:14-168 (same identifiers and values, so native
 * callers compile unchanged and python/audioflux/type/basic.py:25-353 keeps passing the same
 * ints).  Only the enums the hot path consumes are declared.
 */
#ifndef AFB200_TYPES_H
#define AFB200_TYPES_H
#ifdef __cplusplus
extern "C" {
#endif

typedef enum { Window_Rect = 0, Window_Hann, Window_Hamm, Window_Blackman, Window_Kaiser,
               Window_Bartlett, Window_Triang, Window_Flattop, Window_Gauss,
               Window_Blackman_Harris, Window_Blackman_Nuttall, Window_Bartlett_Hann,
               Window_Bohman, Window_Tukey } WindowType;

typedef enum { SpectralData_Power = 0, SpectralData_Mag } SpectralDataType;

typedef enum { SpectralFilterBankScale_Linear = 0, SpectralFilterBankScale_Linspace,
               SpectralFilterBankScale_Mel, SpectralFilterBankScale_Bark,
               SpectralFilterBankScale_Erb, SpectralFilterBankScale_Octave,
               SpectralFilterBankScale_Log, SpectralFilterBankScale_Deep,
               SpectralFilterBankScale_Chroma, SpectralFilterBankScale_LogChroma,
               SpectralFilterBankScale_DeepChroma } SpectralFilterBankScaleType;

typedef enum { SpectralFilterBankStyle_Slaney = 0, SpectralFilterBankStyle_ETSI,
               SpectralFilterBankStyle_Gammatone, SpectralFilterBankStyle_Point,
               SpectralFilterBankStyle_Rect, SpectralFilterBankStyle_Hann,
               SpectralFilterBankStyle_Hamm, SpectralFilterBankStyle_Blackman,
               SpectralFilterBankStyle_Bohman, SpectralFilterBankStyle_Kaiser,
               SpectralFilterBankStyle_Gauss } SpectralFilterBankStyleType;

typedef enum { SpectralFilterBankNormal_None = 0, SpectralFilterBankNormal_Area,
               SpectralFilterBankNormal_BandWidth } SpectralFilterBankNormalType;

typedef enum { ChromaDataNormal_None = 0, ChromaDataNormal_Max, ChromaDataNormal_Min, ChromaDataNormal_P2,
               ChromaDataNormal_P1 } ChromaDataNormalType;

typedef enum { CepstralRectify_Log = 0, CepstralRectify_CubicRoot } CepstralRectifyType;
typedef enum { CepstralEnergy_Replace = 0, CepstralEnergy_Append, CepstralEnergy_Ignore } CepstralEnergyType;

/* src/flux_base.h:103-116 (spectral novelty; "Entroy" is the reference's spelling) */
typedef enum { SpectralNoveltyMethod_Sub = 0, SpectralNoveltyMethod_Entroy, SpectralNoveltyMethod_KL,
               SpectralNoveltyMethod_IS } SpectralNoveltyMethodType;
typedef enum { SpectralNoveltyData_Value = 0, SpectralNoveltyData_Number } SpectralNoveltyDataType;

typedef enum { PaddingPosition_Center = 0, PaddingPosition_Right, PaddingPosition_Left } PaddingPositionType;
typedef enum { PaddingMode_Constant = 0, PaddingMode_Reflect, PaddingMode_Wrap } PaddingModeType;

typedef enum { WaveletContinue_Morse = 0, WaveletContinue_Morlet, WaveletContinue_Bump,
               WaveletContinue_Paul, WaveletContinue_DOG, WaveletContinue_Mexican,
               WaveletContinue_Hermit, WaveletContinue_Ricker } WaveletContinueType;

/* src/reassign_algorithm.h:14-22 */
typedef enum { Reassign_All = 0, Reassign_Fre, Reassign_Time, Reassign_None } ReassignType;

/* include/mir/onset_algorithm.h:13-44: the novelty function of an onset and its parameters ("isPostive" is the
 * reference's spelling) */
typedef enum { Novelty_Flux = 0, Novelty_HFC, Novelty_SD, Novelty_SF, Novelty_MKL, Novelty_PD, Novelty_WPD,
               Novelty_NWPD, Novelty_CD, Novelty_RCD, Novelty_Broadband } NoveltyType;
typedef struct {
    int step;          /* >= 1 */
    float p;           /* != 0 */
    int isPostive;
    int isExp;
    int type;          /* 0 sum, 1 mean */
    float threshold;   /* >= 0 */
    int isNorm;        /* 0 | 1 */
    float gamma;
} NoveltyParam;

#ifdef __cplusplus
}
#endif
#endif
