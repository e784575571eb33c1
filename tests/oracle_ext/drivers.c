/* ORACLE -- TEST INFRASTRUCTURE ONLY. The batch drivers of tests/oracle_ext/oracle_ext.h. */
#include <pthread.h>

#include "oracle_ext.h"

typedef struct { void (*fn)(const void *, uint32_t); const void *ctx; uint32_t lo, hi; } shard_t;

static void *shard_run(void *arg) {
    const shard_t *s = (const shard_t *)arg;
    for (uint32_t i = s->lo; i < s->hi; ++i) s->fn(s->ctx, i);
    return NULL;
}

void sro_shards(uint32_t n, int nthreads, void (*fn)(const void *ctx, uint32_t i), const void *ctx) {
    if (nthreads < 1) nthreads = 1;
    if ((uint32_t)nthreads > n) nthreads = n ? (int)n : 1;
    shard_t *sh = (shard_t *)malloc(sizeof(shard_t) * (size_t)nthreads);
    pthread_t *th = (pthread_t *)malloc(sizeof(pthread_t) * (size_t)nthreads);
    for (int k = 0; k < nthreads; ++k) {
        const shard_t s = {fn, ctx, (uint32_t)((uint64_t)n * k / nthreads), (uint32_t)((uint64_t)n * (k + 1) / nthreads)};
        sh[k] = s;
        if (nthreads > 1) pthread_create(&th[k], NULL, shard_run, &sh[k]);
        else shard_run(&sh[k]);
    }
    for (int k = 0; k < nthreads && nthreads > 1; ++k) pthread_join(th[k], NULL);
    free(sh); free(th);
}

typedef struct {
    const ftr_t *in; const uint8_t *bank; uint32_t n_slot, slot_stride; int check_sign, r; uint32_t *score;
    uint32_t (*pair)(const ftr_t *, const ftr_t *, int);
} scores_t;

static void scores_row(const void *ctx, uint32_t b) {
    const scores_t *j = (const scores_t *)ctx;
    for (uint32_t t = 0; t < j->n_slot; ++t) {
        const ftr_t *mdl = (const ftr_t *)(j->bank + (size_t)t * j->slot_stride);
        j->score[(size_t)b * j->n_slot + t] =
            (j->check_sign && mdl->save_sign != SAVE_MASK) ? DIS_ERR : j->pair(j->in + b, mdl, j->r);
    }
}

void sro_bank_scores(const ftr_t *in, uint32_t B, const uint8_t *bank, uint32_t n_slot, uint32_t slot_stride,
                     int check_sign, int band_r, uint32_t *score, int nthreads,
                     uint32_t (*pair)(const ftr_t *in, const ftr_t *mdl, int r)) {
    const int r = band_r > VV_FRM_MAX - 1 ? VV_FRM_MAX - 1 : band_r;      /* every r >= 118 is the whole matrix */
    const scores_t j = {in, bank, n_slot, slot_stride, check_sign, r, score, pair};
    sro_shards(B, nthreads, scores_row, &j);
}
