/* ORACLE -- TEST INFRASTRUCTURE ONLY. CPU restatement of libspeech_b200's banded DP without the 2:1 length guard
 * (SR_DTW_BAND | SR_DTW_ANY_RATE, include/speech_recog.h): D(i,j) = get_dis(i,j) + min(D(i-1,j), D(i,j-1), D(i-1,j-1))
 * over the band |j - floor(i*M/I)| <= r, score D(I-1,M-1) / (I+M). A plain loop over every cell of the I x M matrix with
 * the band test, sharing no code with the kernels or with the oracle port's sro_dtw_band. tests/test_any_rate.py checks it
 * against the port on every pair within 2:1. Part of oracle/_build/liboracle_ext.so (tests/oracle_ext/oracle_ext.h). */
#include "oracle_ext.h"

#define UNREACHED INT64_MAX

/* D(I-1, M-1) of x (I rows) against y (M rows) at radius r >= 0, or UNREACHED; I, M in 1..119 */
int64_t sro_rate_d(const int16_t *x, int I, const int16_t *y, int M, int r) {
    int64_t D[VV_FRM_MAX][VV_FRM_MAX];
    for (int i = 0; i < I; ++i)
        for (int j = 0; j < M; ++j) {
            D[i][j] = UNREACHED;
            const int64_t c = (int64_t)i * M / I;
            if (llabs((int64_t)j - c) > r) continue;
            int64_t best = UNREACHED;
            if (i == 0 && j == 0) best = 0;
            if (i > 0 && D[i - 1][j] < best) best = D[i - 1][j];
            if (j > 0 && D[i][j - 1] < best) best = D[i][j - 1];
            if (i > 0 && j > 0 && D[i - 1][j - 1] < best) best = D[i - 1][j - 1];
            if (best != UNREACHED) D[i][j] = best + get_dis(x + 12 * i, y + 12 * j);
        }
    return D[I - 1][M - 1];
}

/* the score of one pair: D / (I + M), or DIS_ERR (empty or over-long sets, unreachable end cell); no 2:1 guard */
uint32_t sro_rate(const ftr_t *in, const ftr_t *mdl, int r) {
    const int I = in->frm_num, M = mdl->frm_num;
    if (I == 0 || M == 0 || I > VV_FRM_MAX || M > VV_FRM_MAX) return DIS_ERR;
    const int64_t d = sro_rate_d(in->mfcc_dat, I, mdl->mfcc_dat, M, r);
    return d == UNREACHED ? DIS_ERR : (uint32_t)(d / (I + M));
}

/* score[b][t] of B inputs against n_slot bank slots (sro_bank_scores) */
void sro_rate_batch(const ftr_t *in, uint32_t B, const uint8_t *bank, uint32_t n_slot, uint32_t slot_stride, int check_sign,
                    int band_r, uint32_t *score, int nthreads) {
    sro_bank_scores(in, B, bank, n_slot, slot_stride, check_sign, band_r, score, nthreads, sro_rate);
}
