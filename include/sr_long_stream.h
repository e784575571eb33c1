/* sr_long_stream.h -- live streams of any length on libspeech_b200.so (extension, ABI version 9): S microphones fed in
 * chunks for as long as they run, every segment the long-form VAD finds decided as soon as it closes.
 *
 * The streaming front end of speech_recog.h (sr_streams_*) keeps the reference's fixed capture: at most 65 535 samples and
 * three segments per stream. This pool has neither limit. Its streams carry the calibration, last_sig and the endpoint FSM
 * from push to push, so a word that crosses a chunk boundary is found whole, and one microphone can be heard for hours.
 *
 * Definition.
 *  - Stream: the concatenation of what was pushed to it since its last reset (or since the pool was created).
 *  - Prefix equality: after any push, let n be the stream's sample count. If n >= n_len, or n_len is not a positive
 *    multiple of 240, then
 *      * the events handed out so far for the stream (by pushes and sr_long_streams_fetch) are exactly the closed records
 *        of sr_recognise_long_batch (sr_long.h) on its n-sample prefix, in order;
 *      * open_start (sr_long_streams_state) is the start of that call's trailing open (SR_ST_VAD_FAIL) record, or
 *        SR_SEG_NULL when it has none, and n_closed is the number of its closed records;
 *      * atap is the call's atap.
 *    The batch call is taken with the same n_len and the same initial atap, under the handle's geometry, matcher (any of
 *    sr_set_match's, SR_DTW_BAND | SR_DTW_ANY_RATE and SR_DTW_SYM_P1 included) and bank as they were at the push that closed each segment.
 *    The matcher includes its margin rule SR_DTW_REJECT(q), so an event carries SR_ST_REJECT exactly where that call's record does.
 *  - Frame rule: frame k (samples 80k .. 80k + 159) is evaluated once n > 80k + 160, the long-form VAD's
 *    "i < len - 160". A segment [start, end) is therefore reported by the push after which n >= end + 881. This is one
 *    sample later than sr_streams_*, which reports a segment once n >= end + 880 (its frames run to the capture's end).
 *  - Calibration: while n < n_len, and n_len is a positive multiple of 240, no frame is evaluated; noise_atap runs over
 *    the first n_len samples at the push that completes them. Otherwise the initial atap is used from the first sample
 *    on, as VAD.C:33-36 does.
 *  - Events reuse sr_stream_event: segment is the index among all of the stream's segments since its last reset (no cap
 *    at 3), start / end are sample offsets since that reset; status, frm_num, best_idx, best_dis and cmd are the fields of
 *    the batch call's record. A segment of more than 119 frames (or none) gets SR_ST_MFCC_FAIL and frm_num 0, as there.
 *
 * Limits. 1 <= max_chunk <= 2^20 and n_len <= 65535. A stream holds at most 2^32 - 1 samples. A push that would take any
 * stream past that limit, or one with chunk_len > max_chunk (lens[s] > max_chunk), fails before any stream changes.
 * reset restarts the chosen streams (and drops their queued events) without touching the others.
 *
 * Events are never dropped: what does not fit max_events stays queued, oldest first, for the next push or
 * sr_long_streams_fetch. Two closings of one stream are at least 19 frames apart (11 inactive frames close a segment,
 * then 8 active ones must open the next before it can close), so one push closes at most
 *     E = ceil(F / 19) segments per stream,  F = ceil((max_chunk + c) / 80),
 * with c = n_len when it is a positive multiple of 240 (the push that completes calibration evaluates every frame so far)
 * and c = 0 otherwise. E * n_streams (sr_long_streams_max_events) is always enough for one push.
 *
 * Storage: each stream keeps a ring of R samples, R = max(n_len, 10 561) + max_chunk rounded up to a multiple of 80, and a
 * mirror of the ring's first 9 680 samples behind it, so every decodable segment is contiguous when it is recognised
 * (DESIGN.md, K14). 2 (R + 9 680) bytes per stream, plus about 2.9 kB per event slot.
 *
 * Per push: one read of the chunk (zero-copy when it is pinned host memory, else one staging copy), four kernels (five
 * with a bank), one D2H copy and ONE synchronisation -- as sr_streams_push. A header of its own, as each extension has;
 * the concurrency test's job table covers its entry points like those of every other header. */
#ifndef SR_LONG_STREAM_H_
#define SR_LONG_STREAM_H_
#include "speech_recog.h"

#ifdef __cplusplus
extern "C" {
#endif

#define SR_LONG_STREAM_CHUNK_MAX (1u << 20)   /* largest max_chunk                               */
#define SR_LONG_STREAM_HISTORY   10561u       /* ring history before a chunk, both geometries    */
#define SR_LONG_STREAM_MIRROR    9680u        /* longest decodable segment (GEOM_B, 119 frames)  */

typedef struct sr_long_stream_pool sr_long_stream_pool;
int sr_long_streams_create(sr_handle *h, uint32_t n_streams, uint32_t max_chunk, uint32_t n_len,
                           const atap_tag *atap /* [n_streams] initial, NULL = zeros */, sr_long_stream_pool **out);
int sr_long_streams_destroy(sr_long_stream_pool *p);
/* restart the streams with which[s] != 0 (NULL = all) from atap[s] (NULL = zeros) */
int sr_long_streams_reset(sr_long_stream_pool *p, const uint8_t *which, const atap_tag *atap);
int sr_long_streams_push(sr_long_stream_pool *p, const uint16_t *chunk /* host [n_streams][chunk_stride] */, uint32_t chunk_len,
                         uint32_t chunk_stride, sr_stream_event *events, uint32_t max_events, uint32_t *n_events);
int sr_long_streams_push_ragged(sr_long_stream_pool *p, const uint16_t *chunk, uint32_t chunk_stride,
                                const uint32_t *lens /* [n_streams] samples for each stream, 0 = none */,
                                sr_stream_event *events, uint32_t max_events, uint32_t *n_events);
int sr_long_streams_fetch(sr_long_stream_pool *p, sr_stream_event *events, uint32_t max_events, uint32_t *n_events);
uint32_t sr_long_streams_pending(const sr_long_stream_pool *p);
/* E * n_streams: the most events one push can produce */
uint32_t sr_long_streams_max_events(const sr_long_stream_pool *p);
/* R, the samples of history each stream's ring holds (see Storage above) */
uint32_t sr_long_streams_ring_len(const sr_long_stream_pool *p);
/* per stream, each [n_streams] or NULL: samples received, closed segments, start of the open segment (SR_SEG_NULL: none),
 * atap */
int sr_long_streams_state(sr_long_stream_pool *p, uint32_t *n_recv, uint32_t *n_closed, uint32_t *open_start, atap_tag *atap);

#ifdef __cplusplus
}
#endif
#endif /* SR_LONG_STREAM_H_ */
