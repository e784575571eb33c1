/* sr_long.h -- long-form VAD and per-segment recognition on libspeech_b200.so (extension, ABI version 7): recordings of
 * any length up to 2^27 samples (4.6 h at 8 kHz), every segment VAD finds, one decision per segment.
 *
 * The reference stops at 65 535 samples (VAD's u16 buf_len) and 3 segments (max_vc_con, VAD.C:203-207), because it
 * records a 2 s buffer on an STM32. Its own recordings are longer: a spoken list of ten digits holds ten segments over
 * 75 885 samples. These calls lift both limits and change nothing else.
 *
 * Long-form VAD: the loop of VAD.C:97-218 with max_vc_con removed and a u32 length.
 *  - Frames i = 0, 80, ... while i < len - 160 (no frames for len <= 160).
 *  - last_sig is carried across the whole recording and never reset.
 *  - The four-state FSM is unchanged, so a segment opens at the first of 8 consecutive active frames (start = i - 7*80)
 *    and closes at the first of 11 consecutive inactive ones (end = i - 11*80 + 160).
 *  - After a close the FSM is back in state 0 and keeps looking.
 *  - A segment that is still open when the frames run out is reported with end = SR_SEG_NULL (the reference's NULL end).
 *  - noise_atap runs over the first n_len samples (n_len <= 65535). atap[b] is left as the caller passed it when
 *    n_len % 240 != 0 or n_len > lens[b], as VAD.C:33-36 does.
 *
 * Per-segment decision: spch_recg's decision (main.c:276-295) applied to every segment.
 *  - get_mfcc on [start, end) with vv_frm_max = 119, in the handle's geometry (sr_set_geometry). x[-1] is the real
 *    preceding sample, except that a segment at sample 0 reads mid_val, as in every batched call.
 *  - Then the handle's matcher (sr_set_match: the greedy walk, SR_DTW_BAND with or without SR_DTW_ANY_RATE, or
 *    SR_DTW_SYM_P1) against the bank, the
 *    strict-'<' first-wins argmin, and
 *    cmd = idx / SR_FTR_PER_COMM.
 *  - Status: SR_ST_VAD_FAIL for an unclosed segment, SR_ST_MFCC_FAIL for 0 frames (which includes segments over 119
 *    frames, as in the reference), SR_ST_OK otherwise. best_idx = 0, best_dis = SR_DIS_ERR, cmd = 0 unless SR_ST_OK.
 *  - Under the margin rule SR_DTW_REJECT(q) of the handle's matcher (speech_recog.h), an SR_ST_OK segment the rule turns
 *    down gets SR_ST_REJECT and keeps its best_idx, best_dis and cmd.
 *
 * Recordings are pcm + b*U, with U <= 2^27 and lens[b] <= U (lens NULL: every recording has U samples); no sample at or
 * past lens[b] is read. n_segs[b] is the true segment count; only the first min(n_segs[b], max_segs) records of
 * recording b are written, and nothing else of the segment arrays. max_segs = 0 is valid and counts only.
 * B * max_segs < 2^32. Device workspaces grow to 0.1 B per sample of the staged PCM plus about 2.9 kB per segment slot
 * (B * max_segs, or per group in the host calls).
 *
 * The host-buffer calls stage whole recordings in groups of at most 256 MB of PCM (at least one recording per group)
 * through two device buffers, so the copy of one group overlaps the kernels of the one before; a recording is never
 * split. The _dev forms take device pointers and are asynchronous on the handle's stream, with no host round trip.
 * Timing tags (sr_timing_enable): 11 the block pass (noise_atap and the block summaries, two launches), 12 the segment
 * pass; recognition adds 1 get_mfcc, 2 status, 3 best-init, 4 or 6 the template scan (greedy or banded DP) and 5 the
 * argmin scatter. Not in speech_recog.h, whose entry points a test enumerates; see DESIGN.md section 2. */
#ifndef SR_LONG_H_
#define SR_LONG_H_
#include "speech_recog.h"

#ifdef __cplusplus
extern "C" {
#endif

#define SR_LONG_U_MAX (1u << 27)      /* longest recording: 2^27 samples, 4.6 h at 8 kHz */

typedef struct { uint32_t start, end, status, frm_num, best_idx, best_dis, cmd; } sr_long_seg;
typedef struct {
    atap_tag    *atap;       /* [B] in / out, or NULL                     */
    uint32_t    *n_segs;     /* [B] true segment counts, or NULL          */
    sr_long_seg *segs;       /* [B][max_segs] (NULL allowed when max_segs = 0) */
} sr_long_out;

/* Long-form noise_atap + VAD: atap [B] in / out, n_segs [B], seg_off [B][max_segs][2] start / end sample offsets. */
int sr_vad_long_batch(sr_handle *h, const uint16_t *pcm, uint32_t U, uint32_t B, const uint32_t *lens /* [B] or NULL = U */,
                      uint32_t n_len, uint32_t max_segs, atap_tag *atap, uint32_t *n_segs, uint32_t *seg_off);
/* Long-form VAD, then the per-segment decision on every segment against the handle's bank. */
int sr_recognise_long_batch(sr_handle *h, const uint16_t *pcm, uint32_t U, uint32_t B, const uint32_t *lens,
                            uint32_t n_len, uint32_t max_segs, const sr_long_out *out);
/* The same on device pointers (out and its fields are host structs of device pointers), asynchronous on the handle's
 * stream. lens[b] > U is read as U. */
int sr_vad_long_batch_dev(sr_handle *h, const uint16_t *pcm, uint32_t U, uint32_t B, const uint32_t *lens, uint32_t n_len,
                          uint32_t max_segs, atap_tag *atap, uint32_t *n_segs, uint32_t *seg_off);
int sr_recognise_long_batch_dev(sr_handle *h, const uint16_t *pcm, uint32_t U, uint32_t B, const uint32_t *lens,
                                uint32_t n_len, uint32_t max_segs, const sr_long_out *out_dev);

#ifdef __cplusplus
}
#endif
#endif /* SR_LONG_H_ */
