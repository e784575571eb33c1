/* ORACLE -- TEST INFRASTRUCTURE ONLY. CPU restatement of the alignment calls of libspeech_b200 (sr_dtw_path_batch,
 * sr_average_bank), written from their definitions in include/speech_recog.h. The reference has no DP, so nothing pins
 * these to it (parity unpinned); tests/test_dp_align.py checks this file against plain numpy references and the kernels
 * against this file. Built by __graft_entry__.build() into oracle/_build/liboracle_align.so; the product library never
 * links it. Self-contained: get_dis is restated here (DTW.C:45-62), and the tests check the scores against sro_dtw_band. */
#include <math.h>
#include <pthread.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#define VV_FRM_MAX 119
#define PATH_MAX_PTS 237         /* 2 * VV_FRM_MAX - 1 */
#define DIS_ERR 0xFFFFFFFFu
#define SAVE_MASK 12345

#pragma pack(push, 1)
typedef struct { uint16_t save_sign; uint16_t frm_num; int16_t mfcc_dat[VV_FRM_MAX * 12]; } ftr_t;   /* MFCC.H:18-25 */
#pragma pack(pop)

/* DTW.C:45-62: squared differences summed in u32 (wrapping), float32 square root, truncated */
static uint32_t get_dis(const int16_t *a, const int16_t *b) {
    uint32_t s = 0;
    for (int k = 0; k < 12; ++k) {
        int32_t d = a[k] - b[k];
        s += (uint32_t)d * (uint32_t)d;
    }
    return (uint32_t)sqrtf((float)s);
}

/* The band score of (fin, fmdl) at radius r (D over the band |j - floor(i*M/I)| <= r, D(I-1,M-1) / (I+M)) and, when path
 * is not NULL, its optimal path: from (I-1, M-1) back to (0, 0), at each cell the neighbour with the smallest D, ties to
 * the diagonal, then (i, j-1), then (i-1, j); written forward as (i, j) byte pairs, 0xFF past *len. Rejected pairs (2:1
 * guard, I or M = 0 or > 119, end cell unreachable): DIS_ERR, *len = 0. */
uint32_t sro_dtw_path(const ftr_t *fin, const ftr_t *fmdl, int r, uint8_t *path, uint32_t *len) {
    static const uint64_t INF = UINT64_MAX;
    const int I = fin->frm_num, M = fmdl->frm_num;
    if (path) memset(path, 0xFF, 2 * PATH_MAX_PTS);
    if (len) *len = 0;
    if (r < 0 || I == 0 || M == 0 || I > VV_FRM_MAX || M > VV_FRM_MAX || I > 2 * M || M > 2 * I) return DIS_ERR;
    if (r > VV_FRM_MAX - 1) r = VV_FRM_MAX - 1;          /* every column of every row: the full matrix */
    uint64_t *D = (uint64_t *)malloc(sizeof(uint64_t) * (size_t)I * M);
    for (int i = 0; i < I; ++i) {
        const int c = (int)((int64_t)i * M / I);
        for (int j = 0; j < M; ++j) {
            uint64_t *x = &D[(size_t)i * M + j];
            *x = INF;
            if (j < c - r || j > c + r) continue;
            uint64_t best = 0;
            if (i || j) {
                best = INF;
                if (i && j && D[(size_t)(i - 1) * M + j - 1] < best) best = D[(size_t)(i - 1) * M + j - 1];
                if (j && D[(size_t)i * M + j - 1] < best) best = D[(size_t)i * M + j - 1];
                if (i && D[(size_t)(i - 1) * M + j] < best) best = D[(size_t)(i - 1) * M + j];
                if (best == INF) continue;
            }
            *x = best + get_dis(fin->mfcc_dat + 12 * i, fmdl->mfcc_dat + 12 * j);
        }
    }
    const uint64_t end = D[(size_t)I * M - 1];
    if (end == INF) { free(D); return DIS_ERR; }
    if (path || len) {
        uint8_t rev[2 * PATH_MAX_PTS];
        int i = I - 1, j = M - 1, L = 0;
        for (;;) {
            rev[2 * L] = (uint8_t)i; rev[2 * L + 1] = (uint8_t)j; ++L;
            if (i == 0 && j == 0) break;
            const uint64_t dg = (i && j) ? D[(size_t)(i - 1) * M + j - 1] : INF;
            const uint64_t lf = j ? D[(size_t)i * M + j - 1] : INF;
            const uint64_t up = i ? D[(size_t)(i - 1) * M + j] : INF;
            if (dg <= lf && dg <= up) { --i; --j; }
            else if (lf <= up) --j;
            else --i;
        }
        if (path)
            for (int q = 0; q < L; ++q) { path[2 * q] = rev[2 * (L - 1 - q)]; path[2 * q + 1] = rev[2 * (L - 1 - q) + 1]; }
        if (len) *len = (uint32_t)L;
    }
    free(D);
    return (uint32_t)(end / (uint64_t)(I + M));
}

static int is_member(const ftr_t *f) { return f->save_sign == SAVE_MASK && f->frm_num >= 1 && f->frm_num <= VV_FRM_MAX; }

/* DTW barycentre averaging of group g (K slots from bank + g*K*stride), the definition of sr_average_bank */
static void average_group(const uint8_t *bank, uint32_t stride, uint32_t K, uint32_t g, int r, uint32_t iters,
                          uint8_t *out, uint32_t *score, uint32_t *anchor) {
    const ftr_t *m[32];
    int mem[32], any = 0;
    for (uint32_t k = 0; k < K; ++k) {
        m[k] = (const ftr_t *)(bank + ((size_t)g * K + k) * stride);
        mem[k] = is_member(m[k]);
        any |= mem[k];
    }
    memset(out + (size_t)g * K * stride, 0xFF, (size_t)K * stride);
    for (uint32_t k = 0; k < K; ++k) if (score) score[(size_t)g * K + k] = DIS_ERR;
    if (anchor) anchor[g] = 0xFFFFFFFFu;
    if (!any) return;
    uint64_t best = UINT64_MAX;
    uint32_t a = 0;
    for (uint32_t k = 0; k < K; ++k) {
        if (!mem[k]) continue;
        uint64_t s = 0;
        for (uint32_t l = 0; l < K; ++l)
            if (l != k && mem[l]) s += sro_dtw_path(m[l], m[k], r, NULL, NULL);
        if (s < best) { best = s; a = k; }
    }
    ftr_t C;
    memcpy(&C, m[a], sizeof C);
    const int M = C.frm_num;
    uint8_t path[2 * PATH_MAX_PTS];
    for (uint32_t t = 0; t < iters; ++t) {
        int64_t sum[VV_FRM_MAX * 12];
        int64_t cnt[VV_FRM_MAX];
        memset(sum, 0, sizeof sum); memset(cnt, 0, sizeof cnt);
        int aligned = 0;
        for (uint32_t l = 0; l < K; ++l) {
            if (!mem[l]) continue;
            uint32_t L = 0;
            if (sro_dtw_path(m[l], &C, r, path, &L) == DIS_ERR) continue;
            aligned = 1;
            for (uint32_t q = 0; q < L; ++q) {
                const int i = path[2 * q], j = path[2 * q + 1];
                for (int c = 0; c < 12; ++c) sum[j * 12 + c] += m[l]->mfcc_dat[i * 12 + c];
                ++cnt[j];
            }
        }
        if (!aligned) continue;                            /* C_{t+1} = C_t */
        for (int j = 0; j < M; ++j)
            for (int c = 0; c < 12; ++c) C.mfcc_dat[j * 12 + c] = (int16_t)(sum[j * 12 + c] / cnt[j]);   /* truncating */
    }
    uint8_t *slot = out + (size_t)g * K * stride;
    const uint16_t hdr[2] = {SAVE_MASK, (uint16_t)M};
    memcpy(slot, hdr, 4);
    memcpy(slot + 4, C.mfcc_dat, (size_t)M * 24);
    C.save_sign = SAVE_MASK;
    for (uint32_t k = 0; k < K; ++k)
        if (mem[k] && score) score[(size_t)g * K + k] = sro_dtw_path(m[k], &C, r, NULL, NULL);
    if (anchor) anchor[g] = a;
}

/* ---- batch drivers, contiguous shards over pthreads ---------------------------------------------------------------- */
typedef struct {
    int kind; uint32_t lo, hi;
    const ftr_t *in, *mdl; int r; uint8_t *path; uint32_t *len, *dis;
    const uint8_t *bank; uint32_t stride, K, iters; uint8_t *out; uint32_t *score, *anchor;
} job_t;

static void *job_run(void *arg) {
    job_t *j = (job_t *)arg;
    for (uint32_t p = j->lo; p < j->hi; ++p) {
        if (j->kind == 0)
            j->dis[p] = sro_dtw_path(j->in + p, j->mdl + p, j->r, j->path ? j->path + (size_t)p * 2 * PATH_MAX_PTS : NULL,
                                     j->len ? j->len + p : NULL);
        else
            average_group(j->bank, j->stride, j->K, p, j->r, j->iters, j->out, j->score, j->anchor);
    }
    return NULL;
}

static void run_jobs(const job_t *proto, uint32_t n, int nthreads) {
    if (nthreads < 1) nthreads = 1;
    if ((uint32_t)nthreads > n) nthreads = n ? (int)n : 1;
    job_t *jobs = (job_t *)malloc(sizeof(job_t) * (size_t)nthreads);
    pthread_t *th = (pthread_t *)malloc(sizeof(pthread_t) * (size_t)nthreads);
    for (int k = 0; k < nthreads; ++k) {
        jobs[k] = *proto;
        jobs[k].lo = (uint32_t)((uint64_t)n * k / nthreads);
        jobs[k].hi = (uint32_t)((uint64_t)n * (k + 1) / nthreads);
        if (nthreads > 1) pthread_create(&th[k], NULL, job_run, &jobs[k]);
        else job_run(&jobs[k]);
    }
    for (int k = 0; k < nthreads && nthreads > 1; ++k) pthread_join(th[k], NULL);
    free(jobs); free(th);
}

/* n pairs (in[p], mdl[p]); path [n][237][2] and len [n] may be NULL */
void sro_dtw_path_batch(const ftr_t *in, const ftr_t *mdl, uint32_t n, int r, uint8_t *path, uint32_t *len, uint32_t *dis,
                        int nthreads) {
    job_t j; memset(&j, 0, sizeof j);
    j.kind = 0; j.in = in; j.mdl = mdl; j.r = r; j.path = path; j.len = len; j.dis = dis;
    run_jobs(&j, n, nthreads);
}

/* G groups of K slots; out has the bank's G*K*stride shape; score [G][K] and anchor [G] may be NULL */
void sro_average_bank(const uint8_t *bank, uint32_t stride, uint32_t K, uint32_t G, int r, uint32_t iters, uint8_t *out,
                      uint32_t *score, uint32_t *anchor, int nthreads) {
    job_t j; memset(&j, 0, sizeof j);
    j.kind = 1; j.bank = bank; j.stride = stride; j.K = K; j.r = r; j.iters = iters; j.out = out; j.score = score;
    j.anchor = anchor;
    run_jobs(&j, G, nthreads);
}
