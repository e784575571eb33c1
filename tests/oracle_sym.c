/* ORACLE -- TEST INFRASTRUCTURE ONLY. CPU restatement of the symmetric slope-constrained DP of libspeech_b200
 * (SR_DTW_SYM_P1, include/speech_recog.h): Sakoe & Chiba's symmetric form with P = 1 over SR_DTW_BAND's band, local
 * distance get_dis (DTW.C:45-62). tests/test_sym_match.py checks it against a plain Python cell-level reference and a
 * brute-force enumeration of every P = 1 path. Built by __graft_entry__.build() into oracle/_build/liboracle_sym.so; the
 * product library never links it. */
#include <math.h>
#include <pthread.h>
#include <stdint.h>
#include <stdlib.h>

#define FRM_MAX 119          /* vv_frm_max */
#define DIS_ERR 0xFFFFFFFFu
#define SAVE_MASK 12345u     /* Flash.H: a signed slot */
#define UNREACHED UINT64_MAX

typedef struct { uint16_t save_sign, frm_num; int16_t mfcc_dat[FRM_MAX * 12]; } ftr_t;   /* MFCC.H:18-25 */

/* DTW.C:45-62: the squared differences summed in u32 (wrapping), then a float square root truncated */
uint32_t sro_sym_get_dis(const int16_t *a, const int16_t *b) {
    uint32_t s = 0;
    for (int k = 0; k < 12; ++k) {
        const int32_t e = (int32_t)a[k] - (int32_t)b[k];
        s += (uint32_t)e * (uint32_t)e;
    }
    return (uint32_t)sqrtf((float)s);
}

/* |j - floor(i*M/I)| <= r, inside the I x M matrix */
static int in_band(int i, int j, int I, int M, int r) {
    if (i < 0 || j < 0 || i >= I || j >= M) return 0;
    const int64_t c = (int64_t)i * M / I;
    return llabs((int64_t)j - c) <= r;
}

/* g(I-1, M-1) of x (I rows) against y (M rows) at radius r, or UNREACHED; I, M in 1..119 */
uint64_t sro_sym_g(const int16_t *x, int I, const int16_t *y, int M, int r) {
    static const int mv[3][2] = {{1, 2}, {1, 1}, {2, 1}};                          /* (di, dj) back to the start cell */
    uint64_t g[FRM_MAX][FRM_MAX];
    for (int i = 0; i < I; ++i)
        for (int j = 0; j < M; ++j) {
            g[i][j] = UNREACHED;
            if (!in_band(i, j, I, M, r)) continue;
            const uint64_t d = sro_sym_get_dis(x + 12 * i, y + 12 * j);
            if (i == 0 && j == 0) { g[0][0] = 2 * d; continue; }
            for (int m = 0; m < 3; ++m) {
                const int si = i - mv[m][0], sj = j - mv[m][1];
                if (si < 0 || sj < 0 || g[si][sj] == UNREACHED) continue;
                uint64_t v;
                if (m == 1) v = g[si][sj] + 2 * d;                              /* the diagonal step */
                else {
                    const int ii = si + 1, jj = sj + 1;                         /* (i, j-1) or (i-1, j): one diagonal step on */
                    if (!in_band(ii, jj, I, M, r)) continue;
                    v = g[si][sj] + 2 * (uint64_t)sro_sym_get_dis(x + 12 * ii, y + 12 * jj) + d;
                }
                if (v < g[i][j]) g[i][j] = v;
            }
        }
    return g[I - 1][M - 1];
}

/* the score of one pair: g / (I + M), or DIS_ERR (empty or over-long sets, the 2:1 guard of DTW.C:133, unreachable end) */
uint32_t sro_sym(const ftr_t *in, const ftr_t *mdl, int r) {
    const int I = in->frm_num, M = mdl->frm_num;
    if (I == 0 || M == 0 || I > FRM_MAX || M > FRM_MAX || I > 2 * M || 2 * I < M) return DIS_ERR;
    const uint64_t g = sro_sym_g(in->mfcc_dat, I, mdl->mfcc_dat, M, r);
    return g == UNREACHED ? DIS_ERR : (uint32_t)(g / (uint64_t)(I + M));
}

/* score[b][t] of B inputs against n_slot bank slots of slot_stride bytes over nthreads pthreads; with check_sign a slot
 * whose save_sign is not SAVE_MASK scores DIS_ERR (main.c:283) */
typedef struct {
    const ftr_t *in; const uint8_t *bank; uint32_t n_slot, slot_stride; int check_sign, r; uint32_t *score, lo, hi;
} job_t;
static void *job_run(void *arg) {
    const job_t *j = (const job_t *)arg;
    for (uint32_t b = j->lo; b < j->hi; ++b)
        for (uint32_t t = 0; t < j->n_slot; ++t) {
            const ftr_t *mdl = (const ftr_t *)(j->bank + (size_t)t * j->slot_stride);
            j->score[(size_t)b * j->n_slot + t] =
                (j->check_sign && mdl->save_sign != SAVE_MASK) ? DIS_ERR : sro_sym(j->in + b, mdl, j->r);
        }
    return NULL;
}
void sro_sym_batch(const ftr_t *in, uint32_t B, const uint8_t *bank, uint32_t n_slot, uint32_t slot_stride, int check_sign,
                   int band_r, uint32_t *score, int nthreads) {
    if (nthreads < 1) nthreads = 1;
    if ((uint32_t)nthreads > B) nthreads = B ? (int)B : 1;
    const int r = band_r > FRM_MAX - 1 ? FRM_MAX - 1 : band_r;      /* every r >= 118 is the whole matrix */
    job_t *jobs = (job_t *)malloc(sizeof(job_t) * (size_t)nthreads);
    pthread_t *th = (pthread_t *)malloc(sizeof(pthread_t) * (size_t)nthreads);
    for (int k = 0; k < nthreads; ++k) {
        job_t j = {in, bank, n_slot, slot_stride, check_sign, r, score, (uint32_t)((uint64_t)B * k / nthreads),
                   (uint32_t)((uint64_t)B * (k + 1) / nthreads)};
        jobs[k] = j;
        if (nthreads > 1) pthread_create(&th[k], NULL, job_run, &jobs[k]);
        else job_run(&jobs[k]);
    }
    if (nthreads > 1)
        for (int k = 0; k < nthreads; ++k) pthread_join(th[k], NULL);
    free(jobs); free(th);
}
