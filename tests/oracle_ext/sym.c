/* ORACLE -- TEST INFRASTRUCTURE ONLY. CPU restatement of the symmetric slope-constrained DP of libspeech_b200
 * (SR_DTW_SYM_P1, include/speech_recog.h): Sakoe & Chiba's symmetric form with P = 1 over SR_DTW_BAND's band, local
 * distance get_dis (DTW.C:45-62). tests/test_sym_match.py checks it against a plain Python cell-level reference and a
 * brute-force enumeration of every P = 1 path. Part of oracle/_build/liboracle_ext.so (tests/oracle_ext/oracle_ext.h). */
#include "oracle_ext.h"

/* |j - floor(i*M/I)| <= r, inside the I x M matrix */
static int in_band(int i, int j, int I, int M, int r) {
    if (i < 0 || j < 0 || i >= I || j >= M) return 0;
    const int64_t c = (int64_t)i * M / I;
    return llabs((int64_t)j - c) <= r;
}

/* g(I-1, M-1) of x (I rows) against y (M rows) at radius r, or INF when unreachable; I, M in 1..119 */
uint64_t sro_sym_g(const int16_t *x, int I, const int16_t *y, int M, int r) {
    static const int mv[3][2] = {{1, 2}, {1, 1}, {2, 1}};                          /* (di, dj) back to the start cell */
    uint64_t g[VV_FRM_MAX][VV_FRM_MAX];
    for (int i = 0; i < I; ++i)
        for (int j = 0; j < M; ++j) {
            g[i][j] = INF;
            if (!in_band(i, j, I, M, r)) continue;
            const uint64_t d = get_dis(x + 12 * i, y + 12 * j);
            if (i == 0 && j == 0) { g[0][0] = 2 * d; continue; }
            for (int m = 0; m < 3; ++m) {
                const int si = i - mv[m][0], sj = j - mv[m][1];
                if (si < 0 || sj < 0 || g[si][sj] == INF) continue;
                uint64_t v;
                if (m == 1) v = g[si][sj] + 2 * d;                              /* the diagonal step */
                else {
                    const int ii = si + 1, jj = sj + 1;                         /* (i, j-1) or (i-1, j): one diagonal step on */
                    if (!in_band(ii, jj, I, M, r)) continue;
                    v = g[si][sj] + 2 * (uint64_t)get_dis(x + 12 * ii, y + 12 * jj) + d;
                }
                if (v < g[i][j]) g[i][j] = v;
            }
        }
    return g[I - 1][M - 1];
}

/* the score of one pair: g / (I + M), or DIS_ERR (empty or over-long sets, the 2:1 guard of DTW.C:133, unreachable end) */
uint32_t sro_sym(const ftr_t *in, const ftr_t *mdl, int r) {
    const int I = in->frm_num, M = mdl->frm_num;
    if (I == 0 || M == 0 || I > VV_FRM_MAX || M > VV_FRM_MAX || I > 2 * M || 2 * I < M) return DIS_ERR;
    const uint64_t g = sro_sym_g(in->mfcc_dat, I, mdl->mfcc_dat, M, r);
    return g == INF ? DIS_ERR : (uint32_t)(g / (uint64_t)(I + M));
}

/* score[b][t] of B inputs against n_slot bank slots (sro_bank_scores) */
void sro_sym_batch(const ftr_t *in, uint32_t B, const uint8_t *bank, uint32_t n_slot, uint32_t slot_stride, int check_sign,
                   int band_r, uint32_t *score, int nthreads) {
    sro_bank_scores(in, B, bank, n_slot, slot_stride, check_sign, band_r, score, nthreads, sro_sym);
}
