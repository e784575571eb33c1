/* ORACLE -- TEST INFRASTRUCTURE ONLY. What the CPU restatements of the extension calls (tests/oracle_ext/*.c) share: the
 * reference's record layouts and constants, get_dis, and the batch drivers. __graft_entry__.build() compiles those sources
 * into oracle/_build/liboracle_ext.so; the product library never links it. Only the sources under tests/ include this
 * file: the oracle port (oracle/sr_oracle.c) and the kernels keep their own get_dis, and the tests compare against both. */
#ifndef ORACLE_EXT_H
#define ORACLE_EXT_H
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#define VV_FRM_MAX 119
#define DIS_ERR 0xFFFFFFFFu
#define SAVE_MASK 12345u     /* Flash.H: a signed slot */
#define FTR_PER_COMM 4
#define INF UINT64_MAX

typedef struct { uint16_t save_sign, frm_num; int16_t mfcc_dat[VV_FRM_MAX * 12]; } ftr_t;    /* MFCC.H:18-25 */
typedef struct { uint32_t mid_val; uint16_t n_thl, z_thl; uint32_t s_thl; } atap_t;          /* VAD.H:10-16 */
typedef struct { uint32_t slot, cmd, segment, start, end, dis; } word_t;                     /* sr_conn_word */
typedef struct { uint32_t from, to, cmd_mask; } arc_t;                                       /* sr_gram_arc */

/* DTW.C:45-62: squared differences summed in u32 (wrapping), float32 square root, truncated */
static inline uint32_t get_dis(const int16_t *a, const int16_t *b) {
    uint32_t s = 0;
    for (int k = 0; k < 12; ++k) {
        const int32_t d = (int32_t)a[k] - (int32_t)b[k];
        s += (uint32_t)d * (uint32_t)d;
    }
    return (uint32_t)sqrtf((float)s);
}

/* fn(ctx, i) for every i in [0, n): contiguous shards, one per thread, on the caller's thread when nthreads <= 1 */
void sro_shards(uint32_t n, int nthreads, void (*fn)(const void *ctx, uint32_t i), const void *ctx);

/* score[b][t] = pair(in[b], slot t, min(band_r, 118)) for B inputs against n_slot bank slots of slot_stride bytes; with
 * check_sign a slot whose save_sign is not SAVE_MASK scores DIS_ERR (main.c:283) */
void sro_bank_scores(const ftr_t *in, uint32_t B, const uint8_t *bank, uint32_t n_slot, uint32_t slot_stride,
                     int check_sign, int band_r, uint32_t *score, int nthreads,
                     uint32_t (*pair)(const ftr_t *in, const ftr_t *mdl, int r));
#endif
