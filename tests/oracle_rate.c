/* ORACLE -- TEST INFRASTRUCTURE ONLY. CPU restatement of libspeech_b200's banded DP without the 2:1 length guard
 * (SR_DTW_BAND | SR_DTW_ANY_RATE, include/speech_recog.h): D(i,j) = get_dis(i,j) + min(D(i-1,j), D(i,j-1), D(i-1,j-1))
 * over the band |j - floor(i*M/I)| <= r, score D(I-1,M-1) / (I+M). A plain loop over every cell of the I x M matrix with
 * the band test, sharing no code with the kernels or with the oracle port's sro_dtw_band. tests/test_any_rate.py checks it
 * against the port on every pair within 2:1. Built by __graft_entry__.build() into oracle/_build/liboracle_rate.so; the
 * product library never links it. */
#include <math.h>
#include <pthread.h>
#include <stdint.h>
#include <stdlib.h>

#define FRM_MAX 119          /* vv_frm_max */
#define DIS_ERR 0xFFFFFFFFu
#define SAVE_MASK 12345u     /* Flash.H: a signed slot */
#define UNREACHED INT64_MAX

typedef struct { uint16_t save_sign, frm_num; int16_t mfcc_dat[FRM_MAX * 12]; } ftr_t;   /* MFCC.H:18-25 */

/* DTW.C:45-62: the squared differences summed in u32 (wrapping), then a float square root truncated */
static uint32_t get_dis(const int16_t *a, const int16_t *b) {
    uint32_t s = 0;
    for (int k = 0; k < 12; ++k) {
        const int32_t e = (int32_t)a[k] - (int32_t)b[k];
        s += (uint32_t)e * (uint32_t)e;
    }
    return (uint32_t)sqrtf((float)s);
}

/* D(I-1, M-1) of x (I rows) against y (M rows) at radius r >= 0, or UNREACHED; I, M in 1..119 */
int64_t sro_rate_d(const int16_t *x, int I, const int16_t *y, int M, int r) {
    int64_t D[FRM_MAX][FRM_MAX];
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
    if (I == 0 || M == 0 || I > FRM_MAX || M > FRM_MAX) return DIS_ERR;
    const int64_t d = sro_rate_d(in->mfcc_dat, I, mdl->mfcc_dat, M, r);
    return d == UNREACHED ? DIS_ERR : (uint32_t)(d / (I + M));
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
                (j->check_sign && mdl->save_sign != SAVE_MASK) ? DIS_ERR : sro_rate(j->in + b, mdl, j->r);
        }
    return NULL;
}
void sro_rate_batch(const ftr_t *in, uint32_t B, const uint8_t *bank, uint32_t n_slot, uint32_t slot_stride, int check_sign,
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
