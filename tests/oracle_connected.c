/* ORACLE -- TEST INFRASTRUCTURE ONLY. CPU restatement of the connected-word decoder of libspeech_b200
 * (sr_connected_batch), written from its definition in include/speech_recog.h. The reference decodes one word per segment,
 * so nothing pins this to it (parity unpinned); tests/test_connected.py checks this file against a plain Python cell-level
 * reference and a brute-force minimum over segmentations, and the kernel against this file. Built by
 * __graft_entry__.build() into oracle/_build/liboracle_connected.so; the product library never links it. Self-contained:
 * get_dis is restated here (DTW.C:45-62). */
#include <math.h>
#include <pthread.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#define VV_FRM_MAX 119
#define CONN_FRM_MAX 818
#define SAVE_MASK 12345
#define FTR_PER_COMM 4
#define INF UINT64_MAX

typedef struct { uint32_t slot, cmd, segment, start, end, dis; } word_t;   /* sr_conn_word */

/* DTW.C:45-62: squared differences summed in u32 (wrapping), float32 square root, truncated */
static uint32_t get_dis(const int16_t *a, const int16_t *b) {
    uint32_t s = 0;
    for (int k = 0; k < 12; ++k) {
        int32_t d = a[k] - b[k];
        s += (uint32_t)d * (uint32_t)d;
    }
    return (uint32_t)sqrtf((float)s);
}

/* a cell: its D and the input frame its word started at; a is better than b: smaller D, on equal D the later start */
typedef struct { uint64_t D; uint32_t start; } cell_t;
static int better(cell_t a, cell_t b) { return a.D < b.D || (a.D == b.D && a.D != INF && a.start > b.start); }

/* one sequence x[N][12] against the bank's n_slot slots of `stride` bytes; words[max_words] may be NULL */
void sro_connected(const int16_t *x, uint32_t N, const uint8_t *bank, uint32_t n_slot, uint32_t stride, uint32_t P,
                   uint32_t max_words, word_t *words, uint32_t *n_words, uint64_t *total) {
    *n_words = 0;
    if (total) *total = 0;
    if (N == 0) return;
    uint32_t *M = (uint32_t *)calloc(n_slot ? n_slot : 1, sizeof(uint32_t));
    int any = 0;
    for (uint32_t t = 0; t < n_slot; ++t) {
        uint16_t hdr[2];
        memcpy(hdr, bank + (size_t)t * stride, 4);
        if (hdr[0] == SAVE_MASK && hdr[1] >= 1 && hdr[1] <= VV_FRM_MAX) { M[t] = hdr[1]; any = 1; }
    }
    if (!any) {
        free(M);
        if (total) *total = UINT64_MAX;
        return;
    }
    cell_t *D = (cell_t *)malloc(sizeof(cell_t) * (size_t)n_slot * VV_FRM_MAX);
    for (size_t q = 0; q < (size_t)n_slot * VV_FRM_MAX; ++q) { D[q].D = INF; D[q].start = 0; }
    uint64_t *E = (uint64_t *)malloc(sizeof(uint64_t) * N);
    uint32_t *Eslot = (uint32_t *)malloc(sizeof(uint32_t) * N), *Estart = (uint32_t *)malloc(sizeof(uint32_t) * N);
    uint64_t Eprev = 0;                                   /* E(-1) */
    for (uint32_t i = 0; i < N; ++i) {
        const int16_t *xi = x + (size_t)i * 12;
        E[i] = INF; Eslot[i] = 0; Estart[i] = 0;
        for (uint32_t t = 0; t < n_slot; ++t) {
            if (!M[t]) continue;
            const int16_t *y = (const int16_t *)(bank + (size_t)t * stride + 4);
            cell_t *row = D + (size_t)t * VV_FRM_MAX;     /* D(i-1, t, .) on entry, D(i, t, .) on exit */
            cell_t diag = {INF, 0};                       /* D(i-1, t, j-1) */
            for (uint32_t j = 0; j < M[t]; ++j) {
                const cell_t up = row[j];
                cell_t best = up;
                if (j == 0) {
                    if (Eprev != INF) {
                        const cell_t enter = {Eprev + P, i};
                        if (better(enter, best)) best = enter;
                    }
                } else {
                    if (better(row[j - 1], best)) best = row[j - 1];
                    if (better(diag, best)) best = diag;
                }
                diag = up;
                if (best.D != INF) best.D += get_dis(xi, y + 12 * j);
                row[j] = best;
            }
            const cell_t end = row[M[t] - 1];
            if (end.D < E[i]) { E[i] = end.D; Eslot[i] = t; Estart[i] = end.start; }   /* strict '<': lowest slot */
        }
        Eprev = E[i];
    }
    uint32_t K = 0;
    for (int64_t i = (int64_t)N - 1; i >= 0; i = (int64_t)Estart[i] - 1) ++K;
    uint32_t k = K;
    for (int64_t i = (int64_t)N - 1; i >= 0; i = (int64_t)Estart[i] - 1) {
        const uint32_t st = Estart[i];
        const uint64_t prev = st ? E[st - 1] : 0;
        --k;
        if (words && k < max_words) {
            word_t w = {Eslot[i], Eslot[i] / FTR_PER_COMM, 0, st, (uint32_t)i + 1, (uint32_t)(E[i] - prev - P)};
            words[k] = w;
        }
    }
    *n_words = K;
    if (total) *total = E[N - 1];
    free(M); free(D); free(E); free(Eslot); free(Estart);
}

/* ---- batch driver, contiguous shards over pthreads ----------------------------------------------------------------- */
typedef struct {
    uint32_t lo, hi;
    const int16_t *feat; const uint32_t *frm; uint32_t frm_stride;
    const uint8_t *bank; uint32_t n_slot, stride, P, max_words;
    word_t *words; uint32_t *n_words; uint64_t *total;
} job_t;

static void *job_run(void *arg) {
    job_t *j = (job_t *)arg;
    for (uint32_t b = j->lo; b < j->hi; ++b)
        sro_connected(j->feat + (size_t)b * j->frm_stride * 12, j->frm[b], j->bank, j->n_slot, j->stride, j->P, j->max_words,
                      j->words ? j->words + (size_t)b * j->max_words : NULL, j->n_words + b, j->total ? j->total + b : NULL);
    return NULL;
}

/* B sequences feat[B][frm_stride][12] of frm[b] frames; words [B][max_words] and total [B] may be NULL */
void sro_connected_batch(const int16_t *feat, const uint32_t *frm, uint32_t frm_stride, uint32_t B, const uint8_t *bank,
                         uint32_t n_slot, uint32_t stride, uint32_t P, uint32_t max_words, word_t *words, uint32_t *n_words,
                         uint64_t *total, int nthreads) {
    if (nthreads < 1) nthreads = 1;
    if ((uint32_t)nthreads > B) nthreads = B ? (int)B : 1;
    job_t *jobs = (job_t *)malloc(sizeof(job_t) * (size_t)nthreads);
    pthread_t *th = (pthread_t *)malloc(sizeof(pthread_t) * (size_t)nthreads);
    for (int k = 0; k < nthreads; ++k) {
        job_t j = {(uint32_t)((uint64_t)B * k / nthreads), (uint32_t)((uint64_t)B * (k + 1) / nthreads), feat, frm, frm_stride,
                   bank, n_slot, stride, P, max_words, words, n_words, total};
        jobs[k] = j;
        if (nthreads > 1) pthread_create(&th[k], NULL, job_run, &jobs[k]);
        else job_run(&jobs[k]);
    }
    for (int k = 0; k < nthreads && nthreads > 1; ++k) pthread_join(th[k], NULL);
    free(jobs); free(th);
}
