/* sr_long_grammar.h -- one grammar decode per long recording on libspeech_b200.so (extension, ABI version 8): the
 * connected-word decoder under a finite-state grammar (speech_recog.h, sr_connected_grammar_batch) carried across EVERY
 * segment the long-form VAD (sr_long.h) finds, in a recording of up to 2^27 samples.
 *
 * sr_recognise_connected_grammar_batch decodes one capture of at most 65 535 samples and three segments; the long-form
 * calls find every segment of a recording but decide each segment alone. A spoken list of digits, a phone number or a PIN
 * read with pauses is one word sequence across many pauses: these calls decode it as one.
 *
 * Definition. A recording is a sequence of segments. A segment is DECODABLE when the long-form VAD closed it (end !=
 * SR_SEG_NULL) and its long features have 1 <= F <= SR_CONN_FRM_MAX frames; F follows sr_mfcc_long_batch's frame rule in
 * the handle's geometry, with the same x[-1] rules. The decode is the recurrence of sr_connected_grammar_batch
 * (speech_recog.h) applied to the concatenation of the recording's decodable segments:
 *  - every within-word cell resets to +inf at each decodable segment's first frame; E_s, and with it the grammar state,
 *    carries over;
 *  - a non-decodable segment (left open at the end, 0 frames, more than SR_CONN_FRM_MAX frames) contributes no frames, and
 *    the state carries across it unchanged;
 *  - ties, copies, the trace-back's source-state rule, the totals for N = 0 (0 if state 0 is final, else UINT64_MAX) and
 *    for no accepting path (UINT64_MAX, 0 words), and dis are those of sr_connected_grammar_batch;
 *  - arithmetic is exact in u64: a recording has at most SR_LONG_GRAM_FRM_MAX frames, so every total is below 2^53.
 * A word's segment is its index among ALL of the recording's VAD segments (or, in the kernel-level form, among all of the
 * sequence's segments); start and end are frames relative to that segment.
 * Under the one-state loop grammar the result is sr_connected_batch of each decodable segment alone, joined in order, the
 * totals summed. A recording of <= 65 535 samples whose long-form VAD finds <= 3 segments decodes exactly as
 * sr_recognise_connected_grammar_batch decodes it.
 *
 * Grammar rules (NULL or malformed grammar, more than SR_GRAM_COPY_MAX copies against the handle's bank) are those of
 * sr_connected_grammar_batch; a failing grammar fails the call before anything is written.
 *
 * Timing tags (sr_timing_enable): 13 the decoder (dtw_long_grammar_kernel). The end-to-end call adds 11 and 12 (the
 * long-form VAD) and 1 (get_mfcc of the feature pieces). The decoder launches take consecutive sequences whose records
 * (12 B per frame and grammar state) fit 256 MB; a sequence whose records alone exceed that runs in a launch of its own,
 * with the record workspace grown to fit it: up to 322 MB for a 2^27-sample recording under 16 states.
 * A header of its own, as each extension has; the concurrency test's job table covers its entry points like those of
 * every other header. See DESIGN.md section K13. */
#ifndef SR_LONG_GRAMMAR_H_
#define SR_LONG_GRAMMAR_H_
#include "sr_long.h"

#ifdef __cplusplus
extern "C" {
#endif

#define SR_LONG_GRAM_FRM_MAX 1677720u   /* frames of a 2^27-sample recording: (2^27 - 160) / 80 + 1 */

/* The kernel-level form: B feature sequences over a flat segment table. Sequence b owns segments seq_seg[b] ..
 * seq_seg[b+1] - 1 (seq_seg [B+1] non-decreasing); segment k has seg_frm[k] <= SR_CONN_FRM_MAX frames (0: nothing to
 * decode), its rows at feat + 12 * (seg_frm[0] + ... + seg_frm[k-1]). words [B][max_words] (only the first min(n_words,
 * max_words) records of sequence b are written) and total [B] may be NULL. Fails before writing anything on a segment
 * over SR_CONN_FRM_MAX frames, a sequence over SR_LONG_GRAM_FRM_MAX frames, 2^32 rows or more in all, a NULL n_words
 * with B > 0, or a grammar that fails. */
int sr_connected_grammar_segs_batch(sr_handle *h, const int16_t *feat /* [rows][12] */, const uint32_t *seq_seg /* [B+1] */,
                                    const uint32_t *seg_frm /* [seq_seg[B]] */, uint32_t B, const sr_grammar *g,
                                    uint32_t penalty, uint32_t max_words, sr_conn_word *words, uint32_t *n_words,
                                    uint64_t *total);

/* The end-to-end form: long-form noise_atap and VAD (pcm, U, lens, n_len and atap as in sr_vad_long_batch), the long
 * features of every decodable segment, and one decode per recording under g. Every segment is decoded whatever max_segs
 * is (0 included); max_segs bounds only the per-segment records written. Any output pointer may be NULL; only the first
 * min(n_segs[b], max_segs) segment records and min(n_words[b], max_words) word records of recording b are written.
 * seg_status: SR_ST_OK for a decodable segment, SR_ST_VAD_FAIL for one open at the end, SR_ST_MFCC_FAIL for F = 0 or
 * F > SR_CONN_FRM_MAX. frm_num is F for a decodable segment, else 0. */
typedef struct {
    atap_tag     *atap;        /* [B] in / out, or NULL (noise_atap then starts from zeros) */
    uint32_t     *n_segs;      /* [B] true segment counts                                  */
    uint32_t     *seg_off;     /* [B][max_segs][2] start / end sample                      */
    uint32_t     *frm_num;     /* [B][max_segs]                                            */
    uint8_t      *seg_status;  /* [B][max_segs] SR_ST_*                                    */
    uint32_t     *n_words;     /* [B]                                                      */
    sr_conn_word *words;       /* [B][max_words]                                           */
    uint64_t     *total;       /* [B]                                                      */
} sr_long_gram_out;
int sr_recognise_long_grammar_batch(sr_handle *h, const uint16_t *pcm, uint32_t U, uint32_t B, const uint32_t *lens,
                                    uint32_t n_len, const sr_grammar *g, uint32_t penalty, uint32_t max_segs,
                                    uint32_t max_words, const sr_long_gram_out *out);

#ifdef __cplusplus
}
#endif
#endif /* SR_LONG_GRAMMAR_H_ */
