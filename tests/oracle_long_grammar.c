/* ORACLE -- TEST INFRASTRUCTURE ONLY. CPU restatement of the long-recording grammar decoder of libspeech_b200
 * (sr_connected_grammar_segs_batch, and the one decode per recording of sr_recognise_long_grammar_batch), written from
 * its definition in include/sr_long_grammar.h: sr_connected_grammar_batch's recurrence over the concatenation of a
 * sequence's segments, any number of them, every within-word cell reset at each segment with frames, totals in u64.
 * Nothing pins it to the reference, which decodes one word per segment (parity unpinned); tests/test_long_grammar.py
 * checks this file against a plain Python cell-level reference, against tests/oracle_grammar.c where both apply and
 * against tests/oracle_connected.c under the loop grammar, and the kernel against this file. Built by
 * __graft_entry__.build() into oracle/_build/liboracle_long_grammar.so; the product library never links it.
 * Self-contained: get_dis is restated here (DTW.C:45-62). */
#include <math.h>
#include <pthread.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#define VV_FRM_MAX 119
#define SAVE_MASK 12345
#define FTR_PER_COMM 4
#define INF UINT64_MAX

typedef struct { uint32_t slot, cmd, segment, start, end, dis; } word_t;   /* sr_conn_word */
typedef struct { uint32_t from, to, cmd_mask; } arc_t;                      /* sr_gram_arc */

/* DTW.C:45-62: squared differences summed in u32 (wrapping), float32 square root, truncated */
static uint32_t get_dis(const int16_t *a, const int16_t *b) {
    uint32_t s = 0;
    for (int k = 0; k < 12; ++k) {
        int32_t d = a[k] - b[k];
        s += (uint32_t)d * (uint32_t)d;
    }
    return (uint32_t)sqrtf((float)s);
}

/* a cell: its D and the sequence frame its word started at; a is better than b: smaller D, on equal D the later start */
typedef struct { uint64_t D; uint32_t start; } cell_t;
static int better(cell_t a, cell_t b) { return a.D < b.D || (a.D == b.D && a.D != INF && a.start > b.start); }

/* E_s(i) with the copy and start its word came from */
typedef struct { uint64_t D; uint32_t copy, start; } erec_t;

/* one sequence of n_seg segments, segment k with seg_frm[k] frames (0: nothing to decode), their rows back to back at
 * x[.][12], under the grammar (S states, final mask F, arcs) against the bank's n_slot slots of `stride` bytes. Words carry
 * the segment index among all n_seg segments and segment-relative frames. words[max_words] may be NULL. */
void sro_long_grammar(const int16_t *x, uint32_t n_seg, const uint32_t *seg_frm, const uint8_t *bank, uint32_t n_slot,
                      uint32_t stride, uint32_t S, uint32_t F, uint32_t n_arcs, const arc_t *arcs, uint32_t P, uint32_t max_words,
                      word_t *words, uint32_t *n_words, uint64_t *total) {
    uint64_t N64 = 0;
    for (uint32_t k = 0; k < n_seg; ++k) N64 += seg_frm[k];
    const uint32_t N = (uint32_t)N64;
    *n_words = 0;
    if (total) *total = (F & 1u) ? 0 : UINT64_MAX;
    if (N == 0) return;
    if (total) *total = UINT64_MAX;
    /* the copies: (state, member slot) with an arc into the state carrying the slot's command; state-major, then slot */
    uint32_t n_copy = 0;
    uint32_t *cst = (uint32_t *)malloc(sizeof(uint32_t) * (S * n_slot + 1)), *cslot = (uint32_t *)malloc(sizeof(uint32_t) * (S * n_slot + 1));
    uint32_t *csrc = (uint32_t *)malloc(sizeof(uint32_t) * (S * n_slot + 1)), *cM = (uint32_t *)malloc(sizeof(uint32_t) * (S * n_slot + 1));
    for (uint32_t s = 0; s < S; ++s)
        for (uint32_t t = 0; t < n_slot; ++t) {
            uint16_t hdr[2];
            memcpy(hdr, bank + (size_t)t * stride, 4);
            if (hdr[0] != SAVE_MASK || hdr[1] < 1 || hdr[1] > VV_FRM_MAX) continue;
            uint32_t src = 0;
            for (uint32_t a = 0; a < n_arcs; ++a)
                if (arcs[a].to == s && ((arcs[a].cmd_mask >> (t / FTR_PER_COMM)) & 1u)) src |= 1u << arcs[a].from;
            if (!src) continue;
            cst[n_copy] = s; cslot[n_copy] = t; csrc[n_copy] = src; cM[n_copy] = hdr[1];
            ++n_copy;
        }
    cell_t *D = (cell_t *)malloc(sizeof(cell_t) * ((size_t)n_copy * VV_FRM_MAX + 1));
    erec_t *E = (erec_t *)malloc(sizeof(erec_t) * (size_t)N * S);   /* E[i * S + s] */
    uint32_t *fseg = (uint32_t *)malloc(sizeof(uint32_t) * (size_t)N), *ffirst = (uint32_t *)malloc(sizeof(uint32_t) * (size_t)N);
    uint64_t Eprev[32];                                             /* E_s(i-1) */
    for (uint32_t s = 0; s < S; ++s) Eprev[s] = s == 0 ? 0 : INF;
    uint32_t i = 0;
    for (uint32_t k = 0; k < n_seg; ++k) {
        if (!seg_frm[k]) continue;                                  /* nothing to decode: the state carries across */
        for (size_t q = 0; q < (size_t)n_copy * VV_FRM_MAX; ++q) { D[q].D = INF; D[q].start = 0; }
        const uint32_t first = i;
        for (uint32_t li = 0; li < seg_frm[k]; ++li, ++i) {
            const int16_t *xi = x + (size_t)i * 12;
            fseg[i] = k; ffirst[i] = first;
            for (uint32_t s = 0; s < S; ++s) { E[(size_t)i * S + s].D = INF; E[(size_t)i * S + s].copy = 0; E[(size_t)i * S + s].start = 0; }
            for (uint32_t c = 0; c < n_copy; ++c) {
                const int16_t *y = (const int16_t *)(bank + (size_t)cslot[c] * stride + 4);
                uint64_t ein = INF;                                 /* min over src of E_s(i-1) */
                for (uint32_t s = 0; s < S; ++s)
                    if (((csrc[c] >> s) & 1u) && Eprev[s] < ein) ein = Eprev[s];
                cell_t *row = D + (size_t)c * VV_FRM_MAX;           /* D(i-1, c, .) on entry, D(i, c, .) on exit */
                cell_t diag = {INF, 0};
                for (uint32_t j = 0; j < cM[c]; ++j) {
                    const cell_t up = row[j];
                    cell_t best = up;
                    if (j == 0) {
                        if (ein != INF) {
                            const cell_t enter = {ein + P, i};
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
                const cell_t end = row[cM[c] - 1];
                erec_t *e = &E[(size_t)i * S + cst[c]];
                if (end.D < e->D) { e->D = end.D; e->copy = c; e->start = end.start; }   /* strict '<': lowest copy */
            }
            for (uint32_t s = 0; s < S; ++s) Eprev[s] = E[(size_t)i * S + s].D;
        }
    }
    uint32_t fs = S;
    for (uint32_t s = 0; s < S; ++s)
        if (((F >> s) & 1u) && E[(size_t)(N - 1) * S + s].D != INF && (fs == S || E[(size_t)(N - 1) * S + s].D < E[(size_t)(N - 1) * S + fs].D))
            fs = s;
    if (fs < S) {
        /* trace-back, twice: count, then write in time order */
        for (int pass = 0; pass < 2; ++pass) {
            uint32_t K = *n_words, k = K;
            if (pass == 0) K = 0;
            int64_t i2 = (int64_t)N - 1;
            uint32_t s = fs;
            while (i2 >= 0) {
                const erec_t r = E[(size_t)i2 * S + s];
                uint32_t src = 0;
                uint64_t prev = 0;
                if (r.start) {                                      /* the source state: argmin of E_s(b-1) over src, lowest s */
                    uint64_t bd = INF;
                    for (uint32_t q = 0; q < S; ++q)
                        if (((csrc[r.copy] >> q) & 1u) && E[(size_t)(r.start - 1) * S + q].D < bd) { bd = E[(size_t)(r.start - 1) * S + q].D; src = q; }
                    prev = bd;
                }
                if (pass == 0) ++K;
                else {
                    --k;
                    if (words && k < max_words) {
                        const uint32_t f0 = ffirst[r.start];
                        word_t w = {cslot[r.copy], cslot[r.copy] / FTR_PER_COMM, fseg[r.start], r.start - f0, (uint32_t)i2 + 1 - f0,
                                    (uint32_t)(r.D - prev - P)};
                        words[k] = w;
                    }
                }
                s = src;
                i2 = (int64_t)r.start - 1;
            }
            if (pass == 0) *n_words = K;
        }
        if (total) *total = E[(size_t)(N - 1) * S + fs].D;
    }
    free(cst); free(cslot); free(csrc); free(cM); free(D); free(E); free(fseg); free(ffirst);
}

/* ---- batch driver, contiguous shards over pthreads ----------------------------------------------------------------- */
typedef struct {
    uint32_t lo, hi;
    const int16_t *feat; const uint32_t *seq_seg, *seg_frm; const uint64_t *row;
    const uint8_t *bank; uint32_t n_slot, stride, S, F, n_arcs; const arc_t *arcs; uint32_t P, max_words;
    word_t *words; uint32_t *n_words; uint64_t *total;
} job_t;

static void *job_run(void *arg) {
    job_t *j = (job_t *)arg;
    for (uint32_t b = j->lo; b < j->hi; ++b) {
        const uint32_t k0 = j->seq_seg[b];
        sro_long_grammar(j->feat + j->row[k0] * 12, j->seq_seg[b + 1] - k0, j->seg_frm + k0, j->bank, j->n_slot, j->stride,
                         j->S, j->F, j->n_arcs, j->arcs, j->P, j->max_words,
                         j->words ? j->words + (size_t)b * j->max_words : NULL, j->n_words + b, j->total ? j->total + b : NULL);
    }
    return NULL;
}

/* B sequences over a flat segment table, as sr_connected_grammar_segs_batch takes them: sequence b owns segments
 * seq_seg[b] .. seq_seg[b+1]-1, segment k's seg_frm[k] rows follow those of the segments before it in feat[.][12].
 * words [B][max_words] and total [B] may be NULL */
void sro_long_grammar_batch(const int16_t *feat, const uint32_t *seq_seg, const uint32_t *seg_frm, uint32_t B, const uint8_t *bank,
                            uint32_t n_slot, uint32_t stride, uint32_t S, uint32_t F, uint32_t n_arcs, const arc_t *arcs, uint32_t P,
                            uint32_t max_words, word_t *words, uint32_t *n_words, uint64_t *total, int nthreads) {
    const uint32_t n_seg = B ? seq_seg[B] : 0;
    uint64_t *row = (uint64_t *)malloc(sizeof(uint64_t) * ((size_t)n_seg + 1));
    row[0] = 0;
    for (uint32_t k = 0; k < n_seg; ++k) row[k + 1] = row[k] + seg_frm[k];
    if (nthreads < 1) nthreads = 1;
    if ((uint32_t)nthreads > B) nthreads = B ? (int)B : 1;
    job_t *jobs = (job_t *)malloc(sizeof(job_t) * (size_t)nthreads);
    pthread_t *th = (pthread_t *)malloc(sizeof(pthread_t) * (size_t)nthreads);
    for (int k = 0; k < nthreads; ++k) {
        job_t j = {(uint32_t)((uint64_t)B * k / nthreads), (uint32_t)((uint64_t)B * (k + 1) / nthreads), feat, seq_seg, seg_frm,
                   row, bank, n_slot, stride, S, F, n_arcs, arcs, P, max_words, words, n_words, total};
        jobs[k] = j;
        if (nthreads > 1) pthread_create(&th[k], NULL, job_run, &jobs[k]);
        else job_run(&jobs[k]);
    }
    for (int k = 0; k < nthreads && nthreads > 1; ++k) pthread_join(th[k], NULL);
    free(jobs); free(th); free(row);
}
