/* ORACLE -- TEST INFRASTRUCTURE ONLY. CPU restatement of the long-form VAD of libspeech_b200 (sr_vad_long_batch,
 * include/sr_long.h): the loop of VAD.C:97-218 with max_vc_con removed and a u32 length. tests/test_long.py checks it
 * against a plain Python transcription of that loop, against the port's sro_vad (oracle/sr_oracle.c) and, where
 * oracle/_ref/libref.so is built, against the reference's own VAD on the first 65 535 samples. Built by
 * __graft_entry__.build() into oracle/_build/liboracle_long.so; the product library never links it. The per-segment
 * recognition (sr_recognise_long_batch) is composed in tests/oracle_long.py from this and the port's get_mfcc and dtw. */
#include <pthread.h>
#include <stdint.h>
#include <stdlib.h>

#define FRAME_LEN 160        /* VAD.H:7 */
#define FRAME_MOV 80         /* VAD.H:8 */
#define SEG_NULL 0xFFFFFFFFu /* the NULL end of VAD.C:117-118 */

typedef struct { uint32_t mid_val; uint16_t n_thl; uint16_t z_thl; uint32_t s_thl; } atap_t;   /* VAD.H:10-16 */

/* Frames i = 0, 80, .. while i < len - 160 (VAD.C:121; none for len <= 160). last_sig is carried over the whole
 * recording and never reset (VAD.C:99). The FSM of VAD.C:164-216 is unchanged: v_durmin_f = 8 consecutive active
 * frames open a segment at the first of them, s_durmax_f = 11 consecutive inactive ones close it (VAD.C:72-75); after a
 * close it is back in state 0 and keeps looking (VAD.C:203-207 without the return). Segment k < max_segs goes to
 * seg[2k], seg[2k+1]; one still open when the frames run out keeps end SEG_NULL. Returns the true count. */
uint32_t sro_vad_long(const uint16_t *vc, uint32_t len, const atap_t *atap, uint32_t max_segs, uint32_t *seg) {
    uint32_t last_sig = 0, cur = 0, front = 0, back = 0, n = 0;
    const uint32_t mid = atap->mid_val;
    const uint32_t a_thl = mid + atap->n_thl, b_thl = mid - atap->n_thl;   /* VAD.C:112-113 (u32 wrap) */
    for (uint32_t i = 0; len > FRAME_LEN && i < len - FRAME_LEN; i += FRAME_MOV) {
        uint32_t frm_sum = 0, frm_zero = 0;
        for (uint32_t h = 0; h < FRAME_LEN; ++h) {                  /* VAD.C:126-129 */
            const uint32_t v = vc[i + h];
            frm_sum += v > mid ? v - mid : mid - v;
        }
        for (uint32_t h = 0; h < FRAME_LEN - 1; ++h) {              /* VAD.C:132-157 */
            const uint32_t v = vc[i + h], w = vc[i + h + 1];
            if (v >= a_thl) last_sig = 2; else if (v < b_thl) last_sig = 1;
            if (w >= a_thl) { if (last_sig == 1) ++frm_zero; }
            else if (w < b_thl) { if (last_sig == 2) ++frm_zero; }
        }
        if (frm_sum > atap->s_thl || frm_zero > atap->z_thl) {      /* VAD.C:164-187 */
            if (cur == 0) { cur = 1; front = 1; }
            else if (cur == 1) {
                if (++front >= 8) {
                    cur = 2; front = 0;
                    if (n < max_segs) { seg[2 * n] = i - 7 * FRAME_MOV; seg[2 * n + 1] = SEG_NULL; }
                }
            } else if (cur == 3) { back = 0; cur = 2; }
        } else {                                                    /* VAD.C:188-216 */
            if (cur == 2) { cur = 3; back = 1; }
            else if (cur == 3) {
                if (++back >= 11) {
                    cur = 0; back = 0;
                    if (n < max_segs) seg[2 * n + 1] = i - 11 * FRAME_MOV + FRAME_LEN;
                    ++n;
                }
            } else if (cur == 1) { front = 0; cur = 0; }
        }
    }
    return n + (cur >= 2 ? 1u : 0u);                                 /* + the segment still open */
}

/* B recordings pcm + b*U of lens[b] samples (NULL: U) with atap[b], over nthreads pthreads: n_segs[b] and
 * seg[b][max_segs][2] */
typedef struct {
    const uint16_t *pcm; uint64_t U; const uint32_t *lens; const atap_t *atap; uint32_t max_segs, *n_segs, *seg, lo, hi;
} job_t;
static void *job_run(void *arg) {
    job_t *j = (job_t *)arg;
    for (uint32_t b = j->lo; b < j->hi; ++b)
        j->n_segs[b] = sro_vad_long(j->pcm + (size_t)b * j->U, j->lens ? j->lens[b] : (uint32_t)j->U, j->atap + b, j->max_segs,
                                    j->seg + (size_t)b * 2 * j->max_segs);
    return NULL;
}
void sro_vad_long_batch(const uint16_t *pcm, uint32_t U, uint32_t B, const uint32_t *lens, const atap_t *atap,
                        uint32_t max_segs, uint32_t *n_segs, uint32_t *seg, int nthreads) {
    if (nthreads < 1) nthreads = 1;
    if ((uint32_t)nthreads > B) nthreads = B ? (int)B : 1;
    job_t *jobs = (job_t *)malloc(sizeof(job_t) * (size_t)nthreads);
    pthread_t *th = (pthread_t *)malloc(sizeof(pthread_t) * (size_t)nthreads);
    for (int k = 0; k < nthreads; ++k) {
        job_t j = {pcm, U, lens, atap, max_segs, n_segs, seg, (uint32_t)((uint64_t)B * k / nthreads),
                   (uint32_t)((uint64_t)B * (k + 1) / nthreads)};
        jobs[k] = j;
        if (nthreads > 1) pthread_create(&th[k], NULL, job_run, &jobs[k]);
        else job_run(&jobs[k]);
    }
    if (nthreads > 1)
        for (int k = 0; k < nthreads; ++k) pthread_join(th[k], NULL);
    free(jobs); free(th);
}
