/* sr_synth.h -- deterministic synthetic 8 kHz / 12-bit PCM for benchmarks and tests (SURVEY.md 8d).
 * NOT part of the reference's call surface: it stands in for the ADC capture (Src/BSP/ADC.C) so
 * that the CPU baseline and the GPU path can be fed byte-identical inputs. Integer-only, so the
 * host and device generators produce the same bytes.
 *
 * Utterance `id` of a batch is generated from seed = seed_base + id (splitmix64 parameter stream):
 *   DC level mid in [1900,2200]; background noise: every 80-sample block holds a random-signed
 *   permutation of {0..79}*na/80 (na in [15,60]) -- uniform amplitude with block-constant energy;
 *   samples [0,2400) are noise only (the 300 ms calibration window of main.c:258);
 *   `nwords` words (first start in [2480,3200), length 2000..3600 samples = 250..450 ms, >= 200 ms
 *   gaps): 3..5 harmonics of f0 in [100,250] Hz, Q8 weights, 20 ms raised-cosine ramps, peak
 *   300..1500 LSB, 10 % white-noise (fricative-like) admixture; a word is dropped if fewer than 1040
 *   noise-only samples would follow it; clip to [0,4095]. */
#ifndef SR_SYNTH_H_
#define SR_SYNTH_H_
#include <stddef.h>
#include <stdint.h>
#include "sr_long_stream.h"
#include "sr_long_grammar.h"
#ifdef __cplusplus
extern "C" {
#endif
/* host generator (multi-threaded, no GPU needed): pcm[B][U] */
int sr_synth_pcm_host(uint16_t *pcm, uint32_t U, uint32_t B, uint64_t seed_base, uint32_t nwords);
/* device generator: pcm_dev is device memory on the current device; asynchronous on `cuda_stream` */
int sr_synth_pcm_dev(uint16_t *pcm_dev, uint32_t U, uint32_t B, uint64_t seed_base, uint32_t nwords, void *cuda_stream);
/* synthetic feature structs for the DTW-only configuration (SURVEY.md 8d config 3): frm_num in
 * [fmin,fmax], mfcc ~ clipped +-3000 triangular-ish noise of scale 600 with +400 on c0;
 * out = B structs of `stride` bytes (>= 2860), save_sign = 12345. Host only. */
int sr_synth_ftr_host(void *out, uint32_t stride, uint32_t B, uint64_t seed_base, uint32_t fmin, uint32_t fmax);
/* WAV ingestion (SURVEY 8f-4): RIFF/WAVE PCM, 8-bit unsigned or 16-bit signed, mono or interleaved (channel 0 is
 * taken) -> the 12-bit unsigned ADC codes the path consumes: 16-bit x -> x/16 + 2048 (C truncation), 8-bit
 * x -> (x-128)*16 + 2048. Host only (input adaptation, like the generator above). Returns the number of samples
 * written (<= max_samples), or -1 on a malformed / unsupported file; *sample_rate receives the file's rate. */
long sr_wav_to_adc12(const void *wav, size_t wav_bytes, uint16_t *out, size_t max_samples, uint32_t *sample_rate);
/* Polyphase resampling of 12-bit codes at `rate` to the 8 kHz every other call takes (DESIGN.md section 8). With
 * (L, M) = (8000, rate) / gcd and the rate's odd-length s32 table h[0..N-1] (csrc/sr_resample_taps.h, centre
 * c = (N-1)/2), u[i] = x[i/L] - 2048 when i % L == 0 and i/L < len, else 0 (outside the recording reads as mid-code):
 *   acc[n] = sum_k h[k] * u[n*M + c - k]  (exact in s32),  y[n] = clamp(2048 + ((acc[n] + 2^14) >> 15), 0, 4095),
 *   out_len = ceil(len * L / M), 0 when len = 0. At 8000 Hz, h = {32768}: the output is the input.
 * Recordings are in + b*U_in with len = lens[b] (lens[b] > U_in is read as U_in; lens NULL: U_in); no sample at or past
 * len is read. Output b is out + b*U_out; only out[b][0, out_len) and out_lens[b] (when out_lens is not NULL) are
 * written. All pointers are device (or managed) memory on the current device, 2-byte aligned (lens and out_lens
 * 4-byte). Asynchronous on `cuda_stream` (NULL: the legacy default stream). Returns 0, or -1 with nothing launched on a
 * rate outside SR_RESAMPLE_RATES, U_in > SR_RESAMPLE_U_MAX, U_out < ceil(U_in * L / M) (the longest out_len a
 * recording of U_in samples can have), a NULL or unusable pointer, or a failed launch. B = 0 does nothing. */
#define SR_RESAMPLE_RATES { 8000, 11025, 16000, 22050, 32000, 44100, 48000 }
#define SR_RESAMPLE_U_MAX (1u << 30)   /* longest input: 6.2 h at 48 kHz, more than 2^27 samples (SR_LONG_U_MAX) out */
int sr_resample_adc12_dev(const uint16_t *in /* [B][U_in] 12-bit codes at `rate` */, uint32_t U_in, uint32_t B,
                          const uint32_t *lens /* [B] device, or NULL = U_in */, uint32_t rate,
                          uint16_t *out /* [B][U_out] 12-bit codes at 8 kHz */, uint32_t U_out,
                          uint32_t *out_lens /* [B] device, or NULL */, void *cuda_stream);
/* Live streams at any rate of SR_RESAMPLE_RATES: a pool of sr_long_stream.h whose streams are fed codes at `rate`, each
 * resampled to 8 kHz on the GPU as it arrives (DESIGN.md, K14 at a rate). With (L, M), N and c = (N-1)/2 the rate's as
 * above, a stream that has received n_in input samples since its reset has the 8 kHz stream
 *   n8(n_in) = max(0, ceil((n_in*L - c) / M)) samples long -- exactly the outputs k whose newest input
 *   (k*M + c) / L is below n_in -- holding the first n8(n_in) outputs of sr_resample_adc12_dev on those n_in samples
 *   (inputs before sample 0 read as mid-code). They never change when more input arrives.
 * Everything sr_long_stream.h says holds on that 8 kHz stream with n = n8(n_in): prefix equality with
 * sr_recognise_long_batch (events, open_start, atap), the frame rule, calibration over its first n_len samples, event
 * numbering and the matcher, bank and geometry rules. Every other sr_long_streams_* call takes the pool as it is:
 *  - chunk_len, chunk_stride, lens and max_chunk (1 .. 2^20) count input samples at `rate`; event positions, n_recv
 *    (sr_long_streams_state) and open_start are 8 kHz positions;
 *  - ring_len and max_events follow sr_long_stream.h's formulas with max_chunk replaced by max8 = ceil(max_chunk*L/M),
 *    the most 8 kHz samples one push can complete (n8(a + b) - n8(a) <= ceil(b*L/M));
 *  - a push that would take a stream's input count past 2^32 - 1, or with lens[s] > max_chunk, fails before any stream
 *    changes; a push runs one kernel more than at 8 kHz (five, six with a bank), still with one synchronisation.
 * Refused before anything is allocated: a rate outside SR_RESAMPLE_RATES and every argument sr_long_streams_create
 * refuses. rate = 8000 creates exactly the pool sr_long_streams_create creates. */
int sr_long_streams_create_at_rate(sr_handle *h, uint32_t n_streams, uint32_t max_chunk /* input samples */,
                                   uint32_t n_len /* 8 kHz samples */, const atap_tag *atap /* [n_streams] or NULL */,
                                   uint32_t rate, sr_long_stream_pool **out);
/* Fixed captures at any rate of SR_RESAMPLE_RATES: a pool of speech_recog.h's streaming front end (sr_streams_*) whose
 * streams are fed codes at `rate`, each resampled to 8 kHz on the GPU as it arrives (DESIGN.md, K4 at a rate). With n8
 * as above, a stream that has received n_in input samples since the last reset has the 8 kHz stream of the first
 * n8(n_in) = max(0, ceil((n_in*L - c) / M)) outputs of sr_resample_adc12_dev on those samples.
 * Equivalence: after any sequence of pushes and resets, the pool is indistinguishable from the 8 kHz pool
 * sr_streams_create(h, n_streams, max_samples, n_len) that is handed, at each push, every stream's outputs
 * [n8(before), n8(after)) as one ragged push, under the same handle settings (geometry, matcher, bank) at each push:
 * the same events from every push and from sr_streams_fetch, in the same order, the same sr_streams_pending and the same
 * sr_streams_segments (seg_off and atap). So every rule of the 8 kHz pool applies to the 8 kHz stream: the capture of
 * max_samples samples, the three segments, calibration over its first n_len samples, and positions in 8 kHz samples.
 * As the 8 kHz pool drops the samples that arrive once its capture holds max_samples, this pool drops the 8 kHz outputs
 * past max_samples (they are never computed); the push that brings them is accepted.
 *  - chunk_len, chunk_stride and lens count input samples at `rate`. A push fails before any stream changes when one of
 *    its lengths exceeds max_in = floor(max_samples*M/L), the longest chunk that never completes more than max_samples
 *    8 kHz samples (n8(a + b) - n8(a) <= ceil(b*L/M)), or when it would take a stream's input count past 2^32 - 1;
 *  - sr_streams_reset restarts the input counts and the filter's history too; a push runs one kernel more than at
 *    8 kHz, still with one staging, one D2H copy of the events and one synchronisation;
 *  - the last ceil(c/L) input samples of a capture complete no output until more input arrives (about 2 ms at every
 *    rate): push a few milliseconds of audio after the end of speech so the VAD sees its last frames.
 * Refused before anything is allocated: a rate outside SR_RESAMPLE_RATES and every argument sr_streams_create refuses.
 * rate = 8000 creates exactly the pool sr_streams_create creates (max_in = max_samples, no input-count limit).
 * A group at a rate is sr_stream_group_create with every shard created by sr_streams_create_at_rate; its push, drain and
 * segment rules are unchanged, and chunk and lens are indexed by global stream. */
int sr_streams_create_at_rate(sr_handle *h, uint32_t n_streams, uint32_t max_samples /* 8 kHz */, uint32_t n_len /* 8 kHz */,
                              uint32_t rate, sr_stream_pool **out);
int sr_stream_group_create_at_rate(sr_handle *const *handles, uint32_t n_handles, uint32_t n_streams,
                                   uint32_t max_samples /* 8 kHz */, uint32_t n_len /* 8 kHz */, uint32_t rate,
                                   sr_stream_group **out);
/* The host-buffer long-form calls at any rate of SR_RESAMPLE_RATES (DESIGN.md, long-form calls at a rate): recordings in
 * host memory, rows of U_in codes at `rate` (sr_wav_to_adc12's output, say), resampled to 8 kHz on the GPU group by group.
 * With (L, M) the rate's as above and U8 = ceil(U_in*L/M), recording b has len_b = lens[b] (U_in when lens is NULL) input
 * samples and the 8 kHz recording y_b = the out_len_b = ceil(len_b*L/M) outputs of sr_resample_adc12_dev on them.
 * Equivalence: the call writes exactly what sr_recognise_long_batch (sr_long.h), resp. sr_recognise_long_grammar_batch
 * (sr_long_grammar.h), writes when given the recordings y_b at stride U8 with lens8[b] = out_len_b and the same n_len,
 * initial atap, max_segs, grammar, penalty and max_words, under the handle's geometry, matcher and bank as they are when
 * the call starts: every output field, and nothing else of the caller's memory. Segment offsets, n_len and atap are in
 * 8 kHz samples, as in every other call.
 *  - Staging: whole recordings in groups of at most 256 MB of input at the rate (at least one recording per group) through
 *    the two device buffers of the 8 kHz calls, the copy of one group overlapping the work on the one before. Per group, on
 *    the handle's stream, one K15 launch (timing tag 15) into an 8 kHz group buffer, then the 8 kHz call's per-group work.
 *  - Refused before any copy or launch, with nothing written: a rate outside SR_RESAMPLE_RATES, U_in > SR_RESAMPLE_U_MAX,
 *    U8 > SR_LONG_U_MAX, lens[b] > U_in, and every argument (with U8 and lens8 for U and lens) or grammar the 8 kHz call
 *    refuses.
 * rate = 8000 is the 8 kHz call: the same bytes and launches, no resample launch. */
int sr_recognise_long_batch_at_rate(sr_handle *h, const uint16_t *pcm /* host [B][U_in] at rate */, uint32_t U_in, uint32_t B,
                                    const uint32_t *lens /* host [B] input samples, or NULL = U_in */, uint32_t rate,
                                    uint32_t n_len /* 8 kHz */, uint32_t max_segs, const sr_long_out *out);
int sr_recognise_long_grammar_batch_at_rate(sr_handle *h, const uint16_t *pcm, uint32_t U_in, uint32_t B,
                                            const uint32_t *lens, uint32_t rate, uint32_t n_len, const sr_grammar *g,
                                            uint32_t penalty, uint32_t max_segs, uint32_t max_words,
                                            const sr_long_gram_out *out);
/* The host-buffer capture calls at any rate of SR_RESAMPLE_RATES (DESIGN.md, capture calls at a rate): save_mdl and
 * spch_recg (speech_recog.h) on captures in host memory, rows of U_in codes at `rate`, resampled to 8 kHz on the GPU.
 * With (L, M) the rate's as above and U8 = ceil(U_in*L/M), capture b becomes y_b = the U8 outputs of
 * sr_resample_adc12_dev on its U_in samples (captures have no lens: every y_b is U8 long).
 * Equivalence: the call writes exactly what the 8 kHz call -- sr_recognise_batch, sr_recognise_batch_multi,
 * sr_enrol_batch, sr_recognise_connected_batch, sr_recognise_connected_grammar_batch -- writes when given the captures y_b
 * at stride U8 with the same n_len, initial atap, bank, penalty, grammar and max_words, under the handle's geometry,
 * matcher, lifter and decision rules as they are when the call starts: every output field, and nothing else of the
 * caller's memory. As there, atap is left untouched when n_len % 240 != 0, and only frm_num and the first frm_num rows of
 * a feature struct are written. n_len, seg_off, atap and word frames are in 8 kHz samples, as in every other call.
 *  - sr_recognise_batch_at_rate keeps the 8 kHz call's chunk pipeline and packed transport: chunks of about 32 MB of
 *    input (a multiple of 8 captures), each staged, expanded when packed, then one K15 launch (timing tag 15) and the 8 kHz
 *    recognition of the chunk. sr_transport_stats counts input bytes. sr_recognise_batch_multi_at_rate shards the batch
 *    as sr_recognise_batch_multi does, each shard running sr_recognise_batch_at_rate.
 *  - The other three stage the whole batch in one copy, then one K15 launch (tag 15), then the 8 kHz call's work.
 *  - Refused before any copy or launch, with nothing written: a rate outside SR_RESAMPLE_RATES, U8 > 65535 (so U_in is
 *    at most floor(65535*M/L): 393 210 at 48 kHz, 361 261 at 44.1 kHz, 131 070 at 16 kHz), n_len > U8, and every
 *    argument (with U8 for U), bank or grammar the 8 kHz call refuses.
 * rate = 8000 is the 8 kHz call: the same bytes, launches, tags and transport statistics, no resample launch. */
int sr_recognise_batch_at_rate(sr_handle *h, const uint16_t *pcm /* host [B][U_in] at rate */, uint32_t U_in, uint32_t B,
                               uint32_t rate, uint32_t n_len /* 8 kHz */, const sr_recog_out *out);
int sr_recognise_batch_multi_at_rate(sr_handle *const *handles, uint32_t n_handles, const uint16_t *pcm, uint32_t U_in,
                                     uint32_t B, uint32_t rate, uint32_t n_len, const sr_recog_out *out);
int sr_enrol_batch_at_rate(sr_handle *h, const uint16_t *pcm, uint32_t U_in, uint32_t B, uint32_t rate, uint32_t n_len,
                           void *bank_out, uint32_t slot_stride, uint8_t *status);
int sr_recognise_connected_batch_at_rate(sr_handle *h, const uint16_t *pcm, uint32_t U_in, uint32_t B, uint32_t rate,
                                         uint32_t n_len, uint32_t penalty, uint32_t max_words, const sr_conn_out *out);
int sr_recognise_connected_grammar_batch_at_rate(sr_handle *h, const uint16_t *pcm, uint32_t U_in, uint32_t B, uint32_t rate,
                                                 uint32_t n_len, const sr_grammar *g, uint32_t penalty, uint32_t max_words,
                                                 const sr_conn_out *out);
#ifdef __cplusplus
}
#endif
#endif
