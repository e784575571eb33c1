/* speech_recog.h -- C-ABI of libspeech_b200.so, the H100-native drop-in for the reference's
 * VAD -> MFCC -> DTW hot path (gk969/stm32-speech-recognition, Src/Speech_Recog + the FFT asm).
 *
 * Two layers, both plain C (pointers and sizes only, no CUDA/torch types in any signature):
 *
 *  (1) The reference's own entry points, same names / argument order / struct layouts, each a
 *      batch-of-1 launch of the CUDA kernels on a lazily created default handle (device 0):
 *          noise_atap   Src/Speech_Recog/VAD.H:24   (VAD.C:22-71)
 *          VAD          Src/Speech_Recog/VAD.H:25   (VAD.C:97-218)
 *          get_mfcc     Src/Speech_Recog/MFCC.H:27  (MFCC.C:86-191)
 *          dtw          Src/Speech_Recog/DTW.H:7    (DTW.C:120-192)
 *          fft          Src/Speech_Recog/MFCC.C:27  (global, no header)
 *          get_dis      Src/Speech_Recog/DTW.C:45   (global, no header)
 *          dtw_limit    Src/Speech_Recog/DTW.C:76   (global, no header; its file-static state is per thread here)
 *      A host program written against VAD.H / MFCC.H / DTW.H links unchanged (see include/compat/).
 *
 *  (2) Batched, re-entrant forms on an explicit handle (sr_*): B independent utterances per call,
 *      segments as sample OFFSETS instead of pointers (SR_SEG_NULL = NULL), template bank in the
 *      reference's flash-slot layout (Src/BSP/Flash.H:11-20). Host-buffer variants copy
 *      host->device, launch, copy back and synchronise; *_dev variants take device pointers and
 *      are asynchronous on the handle's stream (sr_set_stream / sr_sync).
 *
 * Results are bit-identical to the reference C compiled for a host CPU (VAD boundaries, MFCC
 * s16, DTW u32 distances, best-template index). There is no CPU fallback: without a CUDA
 * device every compute entry point fails (sr_* return non-zero; the reference-named functions
 * write their failure sentinels and set sr_last_error).
 */
#ifndef SPEECH_RECOG_H_
#define SPEECH_RECOG_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* ---- constants visible through the ABI (same values as the reference's macros) ------------- */
#define SR_FS            8000u        /* ADC.H:7   fs                                   */
#define SR_VCBUF_LEN     16000u       /* ADC.H:9   VcBuf_Len (2 s)                      */
#define SR_ATAP_LEN      2400u        /* ADC.H:11  atap_len (300 ms noise window)       */
#define SR_MAX_VC_CON    3u           /* VAD.H:4   max_vc_con                           */
#define SR_FRAME_LEN     160u         /* VAD.H:7   frame_len (20 ms)                    */
#define SR_FRAME_MOV     80u          /* VAD.H:8   frame_mov (10 ms hop)                */
#define SR_FFT_POINT     1024u        /* MFCC.H:8  fft_point                            */
#define SR_FRQ_MAX       512u         /* MFCC.H:9  frq_max                              */
#define SR_TRI_NUM       24u          /* MFCC.H:12 tri_num                              */
#define SR_MFCC_NUM      12u          /* MFCC.H:13 mfcc_num                             */
#define SR_VV_FRM_MAX    119u         /* MFCC.H:15-16 vv_frm_max                        */
#define SR_DIS_ERR       0xFFFFFFFFu  /* DTW.H:4   dis_err                              */
#define SR_DIS_MAX       0xFFFFFFFFu  /* DTW.H:5   dis_max                              */
#define SR_SAVE_MASK     12345u       /* Flash.H:11 save_mask                           */
#define SR_SIZE_PER_FTR  4096u        /* Flash.H:13 size_per_ftr (flash slot)           */
#define SR_FTR_PER_COMM  4u           /* Flash.H:15 ftr_per_comm                        */
#define SR_COMM_NUM      20u          /* Flash.H:17 comm_num                            */
#define SR_SEG_NULL      0xFFFFFFFFu  /* offset encoding of a NULL valid_tag pointer    */

/* per-utterance status of sr_recognise_* (main.c:38-41: save_ok / VAD_fail / MFCC_fail)       */
#define SR_ST_OK         0u
#define SR_ST_VAD_FAIL   1u
#define SR_ST_MFCC_FAIL  2u
#define SR_ST_REJECT     3u           /* decided, then turned down by the margin rule SR_DTW_REJECT (extension) */

/* ---- the reference's types (VAD.H:10-22, MFCC.H:18-25), identical layout -------------------- */
#ifndef SR_NO_REFERENCE_TYPES
typedef struct {
    uint32_t mid_val;   /* DC level of the capture ("signed zero")           */
    uint16_t n_thl;     /* noise band half-width for the band-crossing rate  */
    uint16_t z_thl;     /* band-crossing-rate threshold                      */
    uint32_t s_thl;     /* short-time magnitude threshold                    */
} atap_tag;

typedef struct {
    uint16_t *start;    /* first sample of the segment (into the caller's PCM buffer) */
    uint16_t *end;      /* one past the last sample; NULL = segment never closed      */
} valid_tag;

#pragma pack(push, 1)
typedef struct {
    uint16_t save_sign;                                   /* SR_SAVE_MASK marks a valid flash template */
    uint16_t frm_num;                                     /* number of MFCC frames                     */
    int16_t  mfcc_dat[SR_VV_FRM_MAX * SR_MFCC_NUM];       /* row-major frame x coefficient             */
} v_ftr_tag;                                              /* 2860 bytes                                */
#pragma pack(pop)
#endif

/* ---- (1) reference-named entry points ------------------------------------------------------- */
void      noise_atap(const uint16_t *noise, uint16_t n_len, atap_tag *atap);
void      VAD(const uint16_t *vc, uint16_t buf_len, valid_tag *valid_voice, atap_tag *atap_arg);
void      get_mfcc(valid_tag *valid, v_ftr_tag *v_ftr, atap_tag *atap_arg);
uint32_t  dtw(v_ftr_tag *ftr_in, v_ftr_tag *frt_mdl);
uint32_t *fft(int16_t *dat_buf, uint16_t buf_len);        /* returns a thread-local u32[1024]; [0,512) valid */
uint32_t  get_dis(int16_t *frm_ftr1, int16_t *frm_ftr2);
uint8_t   dtw_limit(uint16_t x, uint16_t y);            /* DTW.C:76: 0 ins / 1 outs, for the (I,M) of this thread's last dtw() */

/* ---- (2) batched handle API -----------------------------------------------------------------
 * A handle owns its device workspaces and stream; use one handle per thread (calls on the same handle must not
 * overlap). Different handles -- on the same or on different GPUs -- are independent. */
typedef struct sr_handle sr_handle;

int         sr_create(int device, sr_handle **out);       /* device ordinal; <0 = current device     */
int         sr_destroy(sr_handle *h);
/* A handle's device scratch (segments, features, scores, the kernels' utterance hand-out counters) serves ONE stream at a
 * time: sr_sync (or order the new stream behind the old one) before switching streams; concurrent streams take one handle
 * each -- handles are cheap, the tables are per device. */
int         sr_set_stream(sr_handle *h, void *cuda_stream /* cudaStream_t used verbatim; NULL = legacy default stream */);
int         sr_use_own_stream(sr_handle *h);              /* back to the handle's private non-blocking stream (the default) */
int         sr_sync(sr_handle *h);
const char *sr_last_error(const sr_handle *h /* NULL: last error of the calling thread */);
int         sr_device_count(void);                        /* 0 when no CUDA device is usable         */
int         sr_abi_version(void);
void       *sr_host_alloc(size_t bytes);                  /* pinned host memory for fast H2D/D2H     */
void        sr_host_free(void *p);                        /* for sr_host_alloc and sr_host_alloc_dev  */
/* NUMA placement of the host side. The end-to-end call is bound by the H2D copy of the caller's PCM (the u16 v_dat
 * buffer of main.c:249), so on a two-socket box the pinned pages and the threads that feed a GPU belong on the
 * socket that GPU hangs off. sr_host_alloc_dev returns pinned memory whose pages live on `device`'s NUMA node
 * (plain sr_host_alloc on single-node boxes); sr_bind_thread_to_device restricts the CALLING thread (and every
 * thread it creates afterwards, e.g. the library's packer pool) to that node's CPUs and returns the node, or -1 when
 * nothing was changed (one node, unknown topology); sr_device_numa_node / sr_host_numa_node report placement. */
void       *sr_host_alloc_dev(int device, size_t bytes);
int         sr_bind_thread_to_device(int device);
int         sr_device_numa_node(int device);              /* -1 = unknown                            */
int         sr_host_numa_node(const void *p);             /* node backing the page at p; -1 = unknown */

/* Frame geometry of get_mfcc for this handle (sr_mfcc_batch*, sr_recognise_batch*, sr_enrol_batch, streaming):
 *   SR_GEOM_REF  160-sample frames / 80 hop / 1024-point FFT -- the reference's (VAD.H:5-8, MFCC.H:8); bit-exact parity
 *   SR_GEOM_B    200-sample frames / 80 hop /  256-point FFT -- BASELINE configs[0]'s "256-pt/25 ms/10 ms"; an EXTENSION:
 *                the reference's algorithm and Matlab table formulas at the other two sizes, checked only against this
 *                repo's own CPU restatement (parity unpinned by the reference). noise_atap / VAD keep the reference's
 *                framing in both; features of the two geometries must not be mixed in one bank. */
#define SR_GEOM_REF 0
#define SR_GEOM_B   1
int sr_set_geometry(sr_handle *h, int geom);
int sr_get_geometry(const sr_handle *h);

/* Template bank: n_slot slots of slot_stride bytes (>= sizeof(v_ftr_tag), multiple of 4), each
 * starting with a v_ftr_tag; the flash layout of Flash.H:11-20 is slot_stride = 4096.
 * sr_set_bank copies host->device; sr_set_bank_dev borrows a device pointer. */
int sr_set_bank(sr_handle *h, const void *bank, uint32_t n_slot, uint32_t slot_stride);
int sr_set_bank_dev(sr_handle *h, const void *bank_dev, uint32_t n_slot, uint32_t slot_stride);

/* pcm: B utterances, utterance b at pcm + b*U (u16 samples, 12-bit ADC codes).
 * noise_atap over the first n_len samples of every utterance (VAD.C:22-71); atap[b] is left
 * untouched when n_len % 240 != 0 exactly like the reference (VAD.C:33-36). */
int sr_noise_atap_batch(sr_handle *h, const uint16_t *pcm, uint32_t U, uint32_t B, uint32_t n_len,
                        atap_tag *atap /* [B] in/out */);
/* VAD over the first buf_len (<= U) samples; seg_off[b][k][0/1] = start/end offset of segment k */
int sr_vad_batch(sr_handle *h, const uint16_t *pcm, uint32_t U, uint32_t B, uint32_t buf_len,
                 const atap_tag *atap /* [B] */, uint32_t *seg_off /* [B][3][2] */);
/* get_mfcc of one segment per utterance: seg[b*seg_stride + 0/1] = start/end sample offsets.
 * Only frm_num and the first frm_num rows of ftr[b] are written (MFCC.C never writes save_sign); in the host-buffer
 * calls too (this one, sr_recognise_batch*, get_mfcc): save_sign and every row >= frm_num, all rows of a rejected
 * segment (frm_num = 0), come back as the caller passed them.
 * A segment that starts at 0 reads x[-1] = atap[b].mid_val (as a 16-bit sample), not the previous utterance's last
 * sample; every batched entry point does the same (the drop-in get_mfcc reads the caller's start[-1]). */
int sr_mfcc_batch(sr_handle *h, const uint16_t *pcm, uint32_t U, uint32_t B, const uint32_t *seg,
                  uint32_t seg_stride, const atap_tag *atap /* [B] */, v_ftr_tag *ftr /* [B] */);
/* dtw of every input against every bank slot. flags bit0: honour save_sign like spch_recg
 * (main.c:283: slots whose save_sign != 12345 score SR_DIS_ERR). score may be NULL.
 * best_idx/best_dis follow main.c:276-291 (strict '<', first wins, start 0 / 0xFFFFFFFF). */
#define SR_DTW_CHECK_SIGN 1u
#define SR_DTW_BAND       2u          /* use the Sakoe-Chiba banded DP (extension, not in the reference) */
/* With SR_DTW_BAND, band_r is any radius >= 0 (a negative one fails): D(i,j) = get_dis(i,j) + min(D(i-1,j), D(i,j-1),
 * D(i-1,j-1)) over the band |j - floor(i*M/I)| <= band_r, score D(I-1,M-1) / (I+M), SR_DIS_ERR when that cell lies
 * outside the band or the 2:1 length guard of DTW.C:133 rejects the pair. Every band_r >= 118 is the unconstrained DTW
 * over the whole matrix (feature sets have <= 119 frames). Parity unpinned: the reference has no DP; the checker is this
 * project's own CPU restatement. The explicit flags and band_r of sr_dtw_batch decide, never the handle's sr_set_match. */
#define SR_DTW_SYM_P1     4u          /* use the symmetric slope-constrained DP of Sakoe & Chiba (extension, ABI version 10) */
/* With SR_DTW_SYM_P1 (without SR_DTW_BAND: the two together fail before any launch and write nothing), band_r is any
 * radius >= 0 and the band is SR_DTW_BAND's: cell (i, j) is in it iff |j - floor(i*M/I)| <= band_r, every band_r >= 118
 * the whole matrix. With d(i,j) = get_dis(x_i, y_j) (DTW.C:45-62) and 0-based cells, g(0,0) = 2 d(0,0) and
 *   g(i,j) = min(g(i-1,j-2) + 2 d(i,j-1) + d(i,j),  g(i-1,j-1) + 2 d(i,j),  g(i-2,j-1) + 2 d(i-1,j) + d(i,j)),
 * the symmetric form with slope constraint P = 1 (Sakoe & Chiba 1978). A move counts only when its start cell is
 * reachable and every cell it passes through (for a two-step move the intermediate cell and the end cell) lies inside the
 * matrix and the band; any other cell is unreachable ((0,1), for one). Every complete path weighs exactly I + M, so the
 * score g(I-1,M-1) / (I+M) (u32, truncating) is the weighted mean of get_dis along the path. SR_DIS_ERR when the end cell is
 * unreachable, I or M is 0 or above 119, or the 2:1 length guard of DTW.C:133 rejects the pair; SR_DTW_CHECK_SIGN works
 * as with the other matchers. Headroom: g <= (I+M) * 65 536 < 2^24 (get_dis can return 65 536), so 32-bit arithmetic is
 * exact. Parity unpinned: the reference has no DP; the checker is this project's own CPU restatement. */
#define SR_DTW_ANY_RATE   8u          /* SR_DTW_BAND without the 2:1 length guard (extension, ABI version 11) */
/* SR_DTW_BAND | SR_DTW_ANY_RATE (optionally | SR_DTW_CHECK_SIGN) is the SR_DTW_BAND DP above exactly -- the same band
 * |j - floor(i*M/I)| <= band_r, recurrence and score D(I-1,M-1) / (I+M) -- except that the 2:1 length guard of DTW.C:133
 * is not applied, so an utterance spoken at twice or half a template's rate (or faster, or slower) is still scored.
 * SR_DIS_ERR when I or M is 0 or above 119, or when the end cell lies outside the band: for M > I it is ceil(M/I) - 1
 * columns past the band centre of the last row, so a narrow band still rejects extreme ratios, and every band_r >= 118
 * scores every pair of 1..119 frames on both sides. A pair within the guard scores bit for bit what SR_DTW_BAND gives it
 * at the same band_r. SR_DTW_ANY_RATE without SR_DTW_BAND, or with SR_DTW_SYM_P1, fails before any launch and writes
 * nothing. The symmetric P = 1 DP keeps its guard: its slope constraint cannot reach an end cell past 2:1 anyway.
 * Parity unpinned: the reference has no DP; the checker is this project's own CPU restatement. */
#define SR_DTW_REJECT(q)  ((uint32_t)(q) << 16)  /* runner-up margin rule of q per mille (extension, ABI version 12) */
/* SR_DTW_REJECT(q), 1 <= q <= 65535 in bits 16-31 of sr_set_match's flags (q = 0, no bits: no rule), lets a recognition
 * call say "none of these". The reference always names a command (main.c:276-295); the rule applies to each decision it
 * would return, i.e. an utterance or segment whose status is SR_ST_OK. With d1 = best_dis and c1 = cmd as the call returns
 * them and d2 the smallest score over the bank slots t with t / SR_FTR_PER_COMM != c1 (the same scores, save_sign
 * honoured), the decision is rejected iff d2 != SR_DIS_ERR and 1000 * (d2 - d1) < q * d1, computed in 64 bits: the
 * runner-up command is less than q per mille worse than the winner. With no other command, or only SR_DIS_ERR scores
 * there, the decision stands. A rejected record gets status SR_ST_REJECT and keeps best_idx, best_dis, cmd and the scores
 * the call writes without the rule, so a caller can see what was turned down (sr_labels_batch maps it to NULL). The rule
 * goes with every matcher and applies wherever the handle's matcher is read: sr_recognise_batch (both transports), _dev,
 * _dev_allgather (whose gathered keys stay the argmin keys), _multi, the fixed-capture stream pools and groups, the
 * long-recording calls and the live long streams. sr_dtw_batch* have no status to report: any flag bit >= 16 there fails
 * before any copy or launch and writes nothing. */
#define SR_DTW_KNN(k)     ((uint32_t)(k) << 8)   /* K-nearest-neighbour decision rule, 1 <= k <= SR_FTR_PER_COMM (extension) */
/* SR_DTW_KNN(k), 1 <= k <= SR_FTR_PER_COMM in bits 8-10 of sr_set_match's flags (0: no rule), decides by each command's
 * k nearest templates (Rabiner, Levinson, Rosenberg & Wilpon, IEEE TASSP 27(4), 1979) instead of the one nearest slot of
 * main.c:276-292. It applies to an utterance or segment whose status is SR_ST_OK. With s_t the score the call returns for
 * bank slot t (save_sign honoured), command c owns the slots t < n_slot with t / SR_FTR_PER_COMM == c (the last one may
 * own fewer), V_c is the set of its scores that are not SR_DIS_ERR, n_c = |V_c| and m = min(k, n_c): a command with fewer
 * signed templates competes on those it has. Its score is e_c = floor((sum of the m smallest of V_c) / m), the sum in 64
 * bits, and SR_DIS_ERR when n_c = 0. cmd is the command with the smallest e_c (the lowest on ties), best_idx its slot with
 * the smallest score (the lowest on ties, so cmd == best_idx / SR_FTR_PER_COMM) and best_dis = e_cmd; when every e_c is
 * SR_DIS_ERR they are 0, SR_DIS_ERR and 0, as without the rule. The scores, and every record whose status is not SR_ST_OK,
 * are what the call writes without the rule, and the rule rejects nothing by itself. SR_DTW_KNN(1) is the call without
 * the rule, bit for bit. With SR_DTW_REJECT(q) as well, the margin rule takes d1 = e_cmd and d2 = the smallest e_c over
 * the other commands. _dev_allgather gathers best_dis << 32 | best_idx of this decision. The rule applies where the margin
 * rule does; sr_dtw_batch* accept bits 4-15 other than SR_DTW_LIFTER and ignore them. A build without the rule refuses
 * these flags in sr_set_match, which is how a caller detects it. */
#define SR_DTW_LIFTER     (1u << 13)  /* weight the local distance with a bandpass lifter (extension) */
#define SR_DTW_LIFTER_W   { 10, 16, 21, 25, 27, 28, 27, 25, 21, 16, 10, 4 }  /* W[k-1] = round(4 (1 + 6 sin(pi k / 12))) */
/* SR_DTW_LIFTER scores with the raised-sine bandpass lifter w_k = 1 + 6 sin(pi k / 12) of Juang, Rabiner & Wilpon (IEEE
 * TASSP 35(7), 1987) on the cepstra c1..c12, in integers: mfcc_dat coefficient c of a row (c_{c+1}, MFCC.C:173-183)
 * becomes a'_c = sat16(trunc(a_c * W[c] / 16)) with W = SR_DTW_LIFTER_W, the product in 32 bits, the division truncating
 * toward zero and sat16 clamping to [-32768, 32767] (only |a_c| > 18 724 saturates). The scale keeps every liftered value
 * within 1.75x of the original. Under the bit every matcher scores the pair (x, y) exactly as it scores the liftered pair
 * (L(x), L(y)) without it, L applied to every row of the input and of the template; frame counts, save_sign, the 2:1
 * guard, the band, the normalisation and SR_DIS_ERR are unchanged, and get_dis is still the square root of a u32 sum.
 * It combines with each of the four matchers of sr_set_match and with SR_DTW_KNN(k) and SR_DTW_REJECT(q), reaches every
 * recognition call that reads the handle's matcher, and is honoured by sr_dtw_batch*. Enrolment, sr_dtw_path_batch,
 * sr_average_bank, the connected-word and grammar decoders and the drop-in dtw() do not read it. The ABI version stays
 * 12: a build without the lifter refuses the bit in sr_set_match, which is how a caller detects it. */
int sr_dtw_batch(sr_handle *h, const v_ftr_tag *in, uint32_t B, uint32_t flags, int band_r,
                 uint32_t *score /* [B][n_slot] or NULL */, uint32_t *best_idx /* [B] or NULL */,
                 uint32_t *best_dis /* [B] or NULL */);
/* The matcher of this handle's recognition calls: sr_recognise_batch, _dev, _dev_allgather, _multi and every streaming
 * push, each reading it when it starts. flags = 0: the reference's greedy walk (dtw, DTW.C:120-192), the default;
 * flags = SR_DTW_BAND: the banded DP above at radius band_r >= 0 (up to the full matrix); flags = SR_DTW_BAND |
 * SR_DTW_ANY_RATE: the same DP without the 2:1 length guard; flags = SR_DTW_SYM_P1: the
 * symmetric P = 1 DP above at radius band_r >= 0. Recognition keeps honouring save_sign (SR_DTW_CHECK_SIGN, main.c:283)
 * under every matcher. Any other flag value (SR_DTW_SYM_P1 | SR_DTW_BAND and SR_DTW_ANY_RATE alone among them) or a
 * negative band_r fails and leaves the setting unchanged. Each of these four may carry SR_DTW_KNN(k), the KNN rule, and
 * SR_DTW_REJECT(q), the margin rule above, alone or together, and SR_DTW_LIFTER; a KNN field of 5-7 or any other bit in
 * 4-15 fails and leaves the setting unchanged. sr_get_match returns the flags as set, SR_DTW_ANY_RATE, SR_DTW_LIFTER and
 * the rules' bits included. sr_recognise_batch_multi and sr_stream_group_push* fail when their handles have different
 * matchers (with and without SR_DTW_ANY_RATE or SR_DTW_LIFTER differ, and so do different rules);
 * the ranks of an all-gather cannot be checked without a collective, so every rank must set the same one. Enrolment,
 * sr_get_mdl_batch and the drop-in dtw() keep the greedy walk. */
int sr_set_match(sr_handle *h, uint32_t flags, int band_r);
int sr_get_match(const sr_handle *h, uint32_t *flags, int *band_r);
/* spch_recg (main.c:249-296) for B utterances: noise_atap(first n_len) -> VAD(U) -> get_mfcc(seg 0)
 * -> dtw against the bank (the handle's matcher, sr_set_match) -> argmin -> cmd = idx / SR_FTR_PER_COMM. Any output
 * pointer may be NULL. A call writes the fields' [B] records and nothing else of the caller's memory, with two
 * exceptions in every form: atap[b] is left untouched when n_len % 240 != 0, and of ftr[b] only frm_num and its first
 * frm_num rows are written (as sr_mfcc_batch). */
typedef struct {
    atap_tag  *atap;       /* [B]            */
    uint32_t  *seg_off;    /* [B][3][2]      */
    v_ftr_tag *ftr;        /* [B]            */
    uint32_t  *score;      /* [B][n_slot]    */
    uint32_t  *best_idx;   /* [B]            */
    uint32_t  *best_dis;   /* [B] (mtch_dis) */
    uint32_t  *cmd;        /* [B]            */
    uint8_t   *status;     /* [B] SR_ST_*    */
} sr_recog_out;
int sr_recognise_batch(sr_handle *h, const uint16_t *pcm, uint32_t U, uint32_t B, uint32_t n_len,
                       const sr_recog_out *out);

/* Command labels: commstr[] of main.c:25-31, the u8* spch_recg returns (main.c:295). n_labels records of label_stride
 * bytes (the reference: comm_tag {u8 str[3]}), copied. Without a table the reference's own 18 labels are used
 * ("0 ".."9 ", then the GBK codes of up/down/front/back/left/right/big/small). sr_label returns NULL for a command
 * index without a label; sr_labels_batch maps the cmd/status arrays of sr_recognise_batch, NULL where spch_recg
 * returns NULL (VAD or MFCC failed, main.c:261-274). */
int            sr_set_labels(sr_handle *h, const void *labels, uint32_t n_labels, uint32_t label_stride);
const uint8_t *sr_label(const sr_handle *h /* may be NULL: reference table */, uint32_t cmd);
int            sr_labels_batch(const sr_handle *h, const uint32_t *cmd, const uint8_t *status, uint32_t B, const uint8_t **labels_out);

/* The same call spread over several GPUs of one box: contiguous shards, one host thread per handle, results
 * written straight into the caller's host arrays (no collective needed for host outputs). handles[g] must be
 * handles on different devices with the same bank set and the same matcher (sr_set_match). */
int sr_recognise_batch_multi(sr_handle *const *handles, uint32_t n_handles, const uint16_t *pcm, uint32_t U, uint32_t B,
                             uint32_t n_len, const sr_recog_out *out);

/* ---- the one exchange step of the multi-GPU form (SURVEY 8e): NCCL all-gather behind the C-ABI ----------------------
 * Utterances are sharded over ranks -- one handle per GPU, one process or one host thread per rank -- with no
 * data-path communication; at the end the per-template scores (and the 8-byte argmin keys) of all shards are
 * all-gathered. NCCL is bound at run time (dlopen of libnccl.so.2, SR_NCCL_LIB overrides), so single-GPU users need
 * no NCCL at all. sr_comm_unique_id is called on ONE rank and its 128 bytes handed to the others by the host's own
 * means (shared memory between threads, a file, MPI, torch.distributed ...); sr_comm_create is collective.
 * The collective runs on a stream of its own, ordered after the kernels that produced its input, and overlaps whatever
 * the handle's stream does next; sr_comm_wait makes the handle's stream (and thus sr_sync) wait for it. Errors:
 * 10000 + ncclResult_t, or -2 when NCCL cannot be loaded. */
#define SR_COMM_ID_BYTES 128
int sr_comm_unique_id(void *id128);
int sr_comm_create(sr_handle *h, int rank, int world, const void *id128);
int sr_comm_destroy(sr_handle *h);
int sr_comm_rank(const sr_handle *h);
int sr_comm_world(const sr_handle *h);
int sr_comm_nccl_version(void);                           /* 0 when NCCL cannot be loaded */
int sr_comm_wait(sr_handle *h);
int sr_allgather_dev(sr_handle *h, const void *send_dev, void *recv_dev, size_t bytes_per_rank);

/* device-pointer variants: every pointer is device memory on the handle's device, calls are
 * asynchronous on the handle's stream. Alignment: pcm 2 bytes, everything else 4 bytes. */
int sr_noise_atap_batch_dev(sr_handle *h, const uint16_t *pcm, uint32_t U, uint32_t B, uint32_t n_len, atap_tag *atap);
int sr_vad_batch_dev(sr_handle *h, const uint16_t *pcm, uint32_t U, uint32_t B, uint32_t buf_len,
                     const atap_tag *atap, uint32_t *seg_off);
int sr_mfcc_batch_dev(sr_handle *h, const uint16_t *pcm, uint32_t U, uint32_t B, const uint32_t *seg,
                      uint32_t seg_stride, const atap_tag *atap, v_ftr_tag *ftr);
int sr_dtw_batch_dev(sr_handle *h, const v_ftr_tag *in, uint32_t B, uint32_t flags, int band_r,
                     uint32_t *score, uint32_t *best_idx, uint32_t *best_dis);
int sr_recognise_batch_dev(sr_handle *h, const uint16_t *pcm, uint32_t U, uint32_t B, uint32_t n_len,
                           const sr_recog_out *out_dev);
/* sr_recognise_batch_dev on this rank's shard + the exchange step: gathered_score[world*B][n_slot] (rank-major, i.e.
 * global utterance order for equal contiguous shards; needs out_dev->score) and/or gathered_best[world*B] =
 * best_dis << 32 | best_idx, the key of the strict-'<' first-wins argmin (main.c:285-289). Either may be NULL. */
int sr_recognise_batch_dev_allgather(sr_handle *h, const uint16_t *pcm, uint32_t U, uint32_t B, uint32_t n_len,
                                     const sr_recog_out *out_dev, uint32_t *gathered_score, uint64_t *gathered_best);

/* save_mdl (main.c:121-138) for B utterances: noise_atap -> VAD -> get_mfcc(segment 0) -> save_ftr_mdl
 * (Flash.C:17-67) into slot b of a flash-layout bank image bank_out[B][slot_stride] (host memory).
 * status[b] (may be NULL): 0 save_ok / 1 VAD_fail / 2 MFCC_fail; failed slots stay erased (0xFF). */
int sr_enrol_batch(sr_handle *h, const uint16_t *pcm, uint32_t U, uint32_t B, uint32_t n_len, void *bank_out,
                   uint32_t slot_stride, uint8_t *status);
/* get_mdl + get_mean (DTW.C:195-296, defined but never called by the firmware): mdl[p] = element-wise mean of
 * in1[p] and in2[p] along their greedy DTW path, dis[p] = step-normalised path distance; rejected pairs
 * (2:1 length guard) return dis_err and leave mdl[p] untouched. Paths longer than 119 points are truncated
 * (the reference writes out of bounds there). */
int sr_get_mdl_batch(sr_handle *h, const v_ftr_tag *in1, const v_ftr_tag *in2, uint32_t n, v_ftr_tag *mdl, uint32_t *dis);

/* ---- alignment along the banded DP (extension, parity unpinned: the reference has no DP) ---------------------------
 * sr_dtw_path_batch: the SR_DTW_BAND DP of sr_dtw_batch for n (in[p], mdl[p]) pairs, with its optimal warping path.
 * dis[p] equals sr_dtw_batch's band score of the same pair bit for bit. The path is traced back from (I-1, M-1) to (0, 0);
 * at each cell the predecessor is the neighbour with the smallest D, ties to the diagonal (i-1, j-1), then (i, j-1) (only
 * the template advances), then (i-1, j) (only the input advances), so a self-match's path is the diagonal. It is written
 * in forward order as (i, j) byte pairs, path_len[p] = L with max(I, M) <= L <= I + M - 1, entries past L are 0xFF. A
 * rejected pair (2:1 guard, I or M = 0 or > 119, end cell outside the band) has L = 0, all 0xFF and SR_DIS_ERR. path
 * and path_len may be NULL; band_r >= 0 as in sr_dtw_batch (a negative one fails). The handle's sr_set_match is not read. */
#define SR_PATH_MAX 237u   /* 2 * SR_VV_FRM_MAX - 1 */
int sr_dtw_path_batch(sr_handle *h, const v_ftr_tag *in, const v_ftr_tag *mdl, uint32_t n, int band_r,
                      uint8_t *path /* [n][SR_PATH_MAX][2] or NULL */, uint32_t *path_len /* [n] or NULL */,
                      uint32_t *dis /* [n] */);
/* sr_average_bank: one template per group by DTW barycentre averaging. The bank image holds G groups of K consecutive
 * slots (1 <= K <= 32) of slot_stride bytes, e.g. the SR_FTR_PER_COMM repetitions sr_enrol_batch wrote per command. A slot
 * is a member when save_sign == SR_SAVE_MASK and 1 <= frm_num <= 119. The anchor is the member k with the smallest sum
 * over the other members l of the band score S(l -> k) (u64, SR_DIS_ERR counted as 0xFFFFFFFF, lowest k on a tie); C_0 is
 * its features. Each of `iters` updates aligns every member whose score against C_t is not SR_DIS_ERR along its path and
 * sets C_{t+1}[j] = (sum of the member frames aligned to column j) / (their count), per coefficient, truncating toward
 * zero; C keeps the anchor's frame count, and with no member aligned C_{t+1} = C_t. bank_out has the input's shape: slot
 * g*K holds C_iters signed with SR_SAVE_MASK, the group's other K-1 slots are erased (0xFF), so recognition's
 * cmd = idx / SR_FTR_PER_COMM still names the command. A group with no member gets K erased slots and anchor 0xFFFFFFFF.
 * score[g][k] = S(member k -> C_iters), SR_DIS_ERR for a non-member: what sr_dtw_batch(SR_DTW_BAND | SR_DTW_CHECK_SIGN)
 * returns for that slot against bank_out. score and anchor may be NULL. Every pass runs on the device: 2 * iters + 3
 * launches (the anchor scores, an alignment and an update per iteration, the final scores, the packing), fewer when a
 * pass has no pair (K = 1 has no anchor scores). The handle's sr_set_match is not read. */
int sr_average_bank(sr_handle *h, const void *bank, uint32_t slot_stride, uint32_t K, uint32_t G, int band_r,
                    uint32_t iters, void *bank_out, uint32_t *score /* [G][K] or NULL */, uint32_t *anchor /* [G] or NULL */);

/* ---- connected words: one-pass DP over the template bank (extension) ------------------------------------------------
 * sr_mfcc_long_batch: get_mfcc (MFCC.C:86-191) with vv_frm_max replaced by frm_cap (1 <= frm_cap <= SR_CONN_FRM_MAX), in
 * the handle's geometry. With F the frame count of MFCC.C:102, F <= frm_cap writes rows 0..F-1 of feat[b] and
 * frm_num[b] = F; otherwise frm_num[b] = 0 and no row is written. Rows at or past frm_num[b] keep the caller's bytes. NULL
 * segments, and x[-1] = mid_val for a segment that starts at sample 0, behave as in sr_mfcc_batch. Each segment is cut into
 * pieces of at most 119 frames, piece k starting at sample start + 80*119*k, and every piece runs through the get_mfcc
 * kernel; a piece past the first reads its real preceding sample, so every frame is the reference's own frame: pinned to
 * the reference piece by piece. With frm_cap = 119 the result equals sr_mfcc_batch byte for byte. */
#define SR_CONN_FRM_MAX  818u   /* frames of a 65 535-sample segment: (65535 - 160) / 80 + 1 */
#define SR_CONN_SLOT_MAX 128u   /* widest bank sr_connected_batch and sr_recognise_connected_batch accept */
int sr_mfcc_long_batch(sr_handle *h, const uint16_t *pcm, uint32_t U, uint32_t B, const uint32_t *seg, uint32_t seg_stride,
                       const atap_tag *atap /* [B] */, uint32_t frm_cap, int16_t *feat /* [B][frm_cap][12] */,
                       uint32_t *frm_num /* [B] */);
/* sr_connected_batch: the best sequence of words for each of B feature sequences X = x_0..x_{N-1} (N = frm_num[b] <=
 * SR_CONN_FRM_MAX, rows at feat + b*frm_stride*12) against the handle's bank. Members are the slots with save_sign ==
 * SR_SAVE_MASK and 1 <= frm_num <= 119; d(i, t, j) = get_dis(x_i, y_{t,j}) (DTW.C:45-62). With E(-1) = 0 and D(-1,.,.) = inf:
 *   D(i, t, 0)      = d + min(D(i-1, t, 0), E(i-1) + penalty)
 *   D(i, t, j >= 1) = d + min(D(i-1, t, j), D(i, t, j-1), D(i-1, t, j-1))
 *   E(i) = min over members t of D(i, t, M_t - 1),   total = E(N-1)
 * so total = min over segmentations of X and words t_k of the sum of (unnormalised full-matrix DTW + penalty). Ties: every
 * cell carries the input frame its word started at, and takes the predecessor with the smallest D, on equal D the one whose
 * word started later (a new word wins a tie); E(i) ties to the lowest slot (main.c:285-289). The trace-back from frame
 * N-1 gives the words in time order: dis = the word's own path sum (the unnormalised full DTW of its frames against the
 * slot), sum(dis + penalty) = total. n_words[b] is the true count, only the first min(n_words, max_words) records of
 * words[b] are written. N = 0: 0 words, total 0; no member: 0 words, total UINT64_MAX. No band, no 2:1 guard; the handle's
 * sr_set_match is not read. A bank wider than SR_CONN_SLOT_MAX, a frm_num[b] above SR_CONN_FRM_MAX or frm_stride, or a NULL
 * n_words with B > 0 fail the call before anything is written. Parity unpinned: the reference decodes one word per
 * segment; the checker is this project's own CPU restatement. */
typedef struct {
    uint32_t slot, cmd;      /* bank slot of the word; cmd = slot / SR_FTR_PER_COMM (main.c:292)     */
    uint32_t segment;        /* VAD segment it came from (0 in sr_connected_batch)                   */
    uint32_t start, end;     /* input frames [start, end) of that segment                            */
    uint32_t dis;            /* the word's own path sum: unnormalised full-matrix DTW of those frames */
} sr_conn_word;
int sr_connected_batch(sr_handle *h, const int16_t *feat /* [B][frm_stride][12] */, const uint32_t *frm_num /* [B] */,
                       uint32_t frm_stride, uint32_t B, uint32_t penalty, uint32_t max_words,
                       sr_conn_word *words /* [B][max_words] or NULL */, uint32_t *n_words /* [B] */,
                       uint64_t *total /* [B] or NULL */);
/* sr_recognise_connected_batch: noise_atap (first n_len) -> VAD(U) -> sr_mfcc_long_batch features (frm_cap =
 * SR_CONN_FRM_MAX) of EVERY closed segment -> sr_connected_batch of each segment on its own -> the words concatenated in
 * segment order, each keeping its segment. Word boundaries never cross a VAD pause. total = the saturating sum over the
 * decoded segments (0 when none has frames). status follows spch_recg on segment 0: SR_ST_VAD_FAIL if it never closed,
 * SR_ST_MFCC_FAIL if it has 0 frames, SR_ST_OK otherwise; later segments with 0 frames add no words. Any output pointer may
 * be NULL. The call writes the fields' [B] records and nothing else, except that atap[b] is left untouched when
 * n_len % 240 != 0 and only the first min(n_words, max_words) records of words[b] are written. */
typedef struct {
    atap_tag     *atap;      /* [B]                */
    uint32_t     *seg_off;   /* [B][3][2]          */
    uint32_t     *frm_num;   /* [B][3]             */
    uint32_t     *n_words;   /* [B]                */
    sr_conn_word *words;     /* [B][max_words]     */
    uint64_t     *total;     /* [B]                */
    uint8_t      *status;    /* [B] SR_ST_*        */
} sr_conn_out;
int sr_recognise_connected_batch(sr_handle *h, const uint16_t *pcm, uint32_t U, uint32_t B, uint32_t n_len,
                                 uint32_t penalty, uint32_t max_words, const sr_conn_out *out);

/* ---- connected words under a finite-state grammar (extension, ABI version 6) ------------------------------------------
 * A grammar is a nondeterministic finite-state network over commands: n_states states (1 <= n_states <=
 * SR_GRAM_STATE_MAX), state 0 the start state; bit s of final_mask set means state s may end the sequence (final_mask != 0,
 * no bit >= n_states); n_arcs arcs {from, to, cmd_mask}, an arc letting a word whose command c = slot / SR_FTR_PER_COMM has
 * bit c set in cmd_mask lead from `from` to `to` (a bank has at most 128 slots: commands 0..31). No epsilon arcs; arcs may
 * share (from, to) or overlap.
 * A COPY is a pair (state s', member slot t) such that some arc into s' carries cmd(t); members as in sr_connected_batch
 * (signed, 1 <= frm_num <= 119). Copies are numbered state-major, then by slot; src(c) is the set of states s with an arc
 * s -> s' carrying cmd(t). At most SR_GRAM_COPY_MAX copies. With E_s(-1) = 0 for s = 0 and +inf otherwise, D(-1,.,.) = inf
 * and d = get_dis (DTW.C:45-62):
 *   D(i, c, 0)      = d + min(D(i-1, c, 0), min_{s in src(c)} E_s(i-1) + penalty)
 *   D(i, c, j >= 1) = d + min(D(i-1, c, j), D(i, c, j-1), D(i-1, c, j-1))
 *   E_s'(i) = min over copies c of state s' of D(i, c, M_t - 1),   total = min over final states s of E_s(N-1)
 * Ties as in sr_connected_batch: cells prefer the later word start, E_s ties to the lowest copy (within a state the lowest
 * slot), the final state ties to the lowest state. Trace-back from the chosen final state at N-1: its record gives (copy
 * c, start b); the word's source state is the argmin over s in src(c) of E_s(b-1) (D only, ties to the lowest s; state 0
 * at b = 0). Words in time order, dis = E(end-1) - E_src(b-1) - penalty. N = 0: 0 words, total 0 if state 0 is final,
 * else UINT64_MAX. No accepting path: 0 words, total UINT64_MAX. The one-state loop grammar (n_states 1, final_mask 1, one
 * arc 0 -> 0 carrying every command) is exactly sr_connected_batch. */
#define SR_GRAM_STATE_MAX 16u
#define SR_GRAM_COPY_MAX  128u   /* = SR_CONN_SLOT_MAX: one decoder warp per copy */
typedef struct { uint32_t from, to, cmd_mask; } sr_gram_arc;
typedef struct { uint32_t n_states, final_mask, n_arcs; const sr_gram_arc *arcs; } sr_grammar;
/* sr_connected_grammar_batch: sr_connected_batch under grammar g, with its argument rules and footprint (only the first
 * min(n_words, max_words) records of words[b] are written), plus B * frm_stride < 2^32 (feature rows are 32-bit
 * indices; the limit is 96 GB of features). A grammar without copies against the bank (no arcs, or arcs whose commands
 * have no member) is valid: 0 words, total as for N = 0 or no accepting path. A NULL or malformed grammar (state count, final mask, an arc
 * endpoint >= n_states, NULL arcs with n_arcs > 0) fails the call, and so does a grammar with more than SR_GRAM_COPY_MAX
 * copies against the handle's bank, whose membership is read from the bank (device memory, 4 header bytes per slot) when
 * the call runs: before any launch and before any caller byte is written. B = 0 launches nothing. */
int sr_connected_grammar_batch(sr_handle *h, const int16_t *feat /* [B][frm_stride][12] */, const uint32_t *frm_num /* [B] */,
                               uint32_t frm_stride, uint32_t B, const sr_grammar *g, uint32_t penalty, uint32_t max_words,
                               sr_conn_word *words /* [B][max_words] or NULL */, uint32_t *n_words /* [B] */,
                               uint64_t *total /* [B] or NULL */);
/* sr_recognise_connected_grammar_batch: noise_atap -> VAD -> long features of every closed segment, as
 * sr_recognise_connected_batch, then ONE decode per capture under g: the capture's segments with frames are one sequence,
 * their frames back to back, and at the first frame of a later segment every within-word cell is reset to +inf, so no word
 * crosses a pause while E, and with it the grammar state, carries over. Words keep their segment and segment-relative
 * start / end. status, atap and the footprint are those of sr_recognise_connected_batch; the grammar rules are those of
 * sr_connected_grammar_batch. Under the loop grammar the result equals sr_recognise_connected_batch bit for bit. */
int sr_recognise_connected_grammar_batch(sr_handle *h, const uint16_t *pcm, uint32_t U, uint32_t B, uint32_t n_len,
                                         const sr_grammar *g, uint32_t penalty, uint32_t max_words, const sr_conn_out *out);

/* ---- streaming front end (stands in for record(), main.c:77-102 / ADC.C:11-103) ----------------------------
 * n_streams concurrent captures of max_samples samples each, fed in chunks -- in lock step (sr_streams_push) or every
 * stream at its own pace (sr_streams_push_ragged). Each push advances noise_atap (once the first n_len samples of a
 * stream are in) and VAD with the reference's carried state, and recognises every segment that closes (get_mfcc + dtw
 * with the handle's matcher + argmin against the handle's bank): one H2D copy, five kernels, one D2H copy and ONE
 * synchronisation per push.
 * After the last chunk the events equal the batch results on the complete buffers; the reference itself only ever
 * recognises segment 0 (main.c:268), here all <= 3 segments of a stream produce an event.
 * Events are never dropped: what does not fit max_events stays queued (oldest first) and is handed out by the next
 * push or by sr_streams_fetch; 3 * n_streams is always enough for one push. */
typedef struct sr_stream_pool sr_stream_pool;
typedef struct {
    uint32_t stream, segment;   /* which stream, which of its <= 3 segments       */
    uint32_t start, end;        /* sample offsets of the segment                   */
    uint32_t status;            /* SR_ST_OK or SR_ST_MFCC_FAIL                     */
    uint32_t frm_num, best_idx, best_dis, cmd;
} sr_stream_event;
int sr_streams_create(sr_handle *h, uint32_t n_streams, uint32_t max_samples, uint32_t n_len, sr_stream_pool **out);
int sr_streams_destroy(sr_stream_pool *p);
int sr_streams_reset(sr_stream_pool *p);
int sr_streams_push(sr_stream_pool *p, const uint16_t *chunk /* host [n_streams][chunk_stride] */, uint32_t chunk_len,
                    uint32_t chunk_stride, sr_stream_event *events, uint32_t max_events, uint32_t *n_events);
int sr_streams_push_ragged(sr_stream_pool *p, const uint16_t *chunk /* host [n_streams][chunk_stride] */, uint32_t chunk_stride,
                           const uint32_t *lens /* [n_streams] samples for each stream, 0 = none */,
                           sr_stream_event *events, uint32_t max_events, uint32_t *n_events);
int sr_streams_fetch(sr_stream_pool *p, sr_stream_event *events, uint32_t max_events, uint32_t *n_events);
uint32_t sr_streams_pending(const sr_stream_pool *p);
int sr_streams_segments(sr_stream_pool *p, uint32_t *seg_off /* [n_streams][3][2] or NULL */, atap_tag *atap /* or NULL */);

/* The same over several GPUs of one box (BASELINE configs[4]): streams [S*g/G, S*(g+1)/G) live on handles[g]; one
 * persistent host thread per shard (bound to its GPU's NUMA node) runs that shard's push, so the G pushes overlap.
 * chunk / lens / seg_off / atap are indexed by GLOBAL stream number, events carry global stream numbers.
 * A group has no fetch or pending call: events that do not fit max_events stay queued on their shard and come out with
 * the group's next push (oldest first, shard after shard); a push of zero samples drains them. */
typedef struct sr_stream_group sr_stream_group;
int sr_stream_group_create(sr_handle *const *handles, uint32_t n_handles, uint32_t n_streams, uint32_t max_samples,
                           uint32_t n_len, sr_stream_group **out);
int sr_stream_group_destroy(sr_stream_group *g);
int sr_stream_group_reset(sr_stream_group *g);
int sr_stream_group_push(sr_stream_group *g, const uint16_t *chunk, uint32_t chunk_len, uint32_t chunk_stride,
                         sr_stream_event *events, uint32_t max_events, uint32_t *n_events);
int sr_stream_group_push_ragged(sr_stream_group *g, const uint16_t *chunk, uint32_t chunk_stride, const uint32_t *lens,
                                sr_stream_event *events, uint32_t max_events, uint32_t *n_events);
int sr_stream_group_segments(sr_stream_group *g, uint32_t *seg_off, atap_tag *atap);

/* secondary globals of the reference, batched: fft magnitudes (MFCC.C:27-62) of n frames of
 * `len` (<=1024) s16 samples each -> u32[n][512]; get_dis (DTW.C:45-62) of n row pairs. */
int sr_fft_mag_batch(sr_handle *h, const int16_t *frames, uint32_t len, uint32_t n, uint32_t *mag);
int sr_get_dis_batch(sr_handle *h, const int16_t *a, const int16_t *b, uint32_t n, uint32_t *dis);
/* dtw_limit (DTW.C:76-109) for n points with explicit frame counts: out[i] = 0 ins / 1 outs */
int sr_dtw_limit_batch(sr_handle *h, const uint16_t *x, const uint16_t *y, const uint16_t *I, const uint16_t *M, uint32_t n,
                       uint8_t *out);
/* raw cr4_fft_1024_stm32 (Src/BSP/cr4_fft_1024_stm32.s:219-281) of n packed inputs (re | im<<16,
 * u32[n][1024]) -> packed outputs; exists so tests can pin the FFT kernel code against the asm restatement
 * on arbitrary complex data */
int sr_fft_raw_batch(sr_handle *h, const uint32_t *in_packed, uint32_t n, uint32_t *out_packed);
/* test hook: the radix-4 FFT device code the MFCC kernels share, alone, at N = 256 (the GEOM_B FFT) or N = 1024, on n
 * packed N-point inputs (u32[n][N]) -> packed outputs; lets tests drive the 256-point FFT with complex, full-length
 * data, which the GEOM_B front end never feeds it. N must be 256 or 1024. */
int sr_debug_fft_raw_n(sr_handle *h, const uint32_t *in_packed, uint32_t N, uint32_t n, uint32_t *out_packed);

/* test hook: count of float bit patterns in [lo_bits, hi_bits) where the kernels' branch-free sqrt differs
 * from the IEEE sqrt.rn.f32 (0 over [1.0f, 2^33), the range the path can produce) */
int sr_debug_sqrt_mismatches(sr_handle *h, uint32_t lo_bits, uint32_t hi_bits, uint64_t *mismatches);
/* test hook: count of v in [lo, hi) (hi <= 2^32) where the MFCC kernels' log100 (a float estimate and two correction
 * loops) differs from a binary search over the same threshold table (0 over [0, 2^32)) */
int sr_debug_log100_mismatches(sr_handle *h, uint64_t lo, uint64_t hi, uint64_t *mismatches);
/* test hook: count of (re, im) pairs of index [lo, hi) where the MFCC kernels' magnitude step differs from
 * (u32)(sqrtf((float)pw) * 10), pw = re^2 + im^2 as an s32, 0 for pw <= 0. which = 0: mag10_small over |re|, |im| <= 8209,
 * index (re + 8209) * 16419 + im + 8209 < 16419^2; which = 1: mag10 over every s16 pair, index (u16)re | (u16)im << 16
 * < 2^32 (0 over each whole domain) */
int sr_debug_mag10_mismatches(sr_handle *h, int which, uint64_t lo, uint64_t hi, uint64_t *mismatches);

/* Packed PCM transport of sr_recognise_batch (host buffers): chunks whose samples are all < 4096 (the reference's
 * 12-bit ADC range) may cross PCIe as 12 bits per sample, packed by host worker threads and expanded on the
 * device; chunks with any larger sample travel as plain u16, so results never change. The caller's thread keeps
 * sending plain chunks from the front of the batch while the workers pack from the back, so the call is never slower
 * than the plain transport and approaches 3/4 of its PCIe time as the CPU share grows. mode: 0 off, 1 on,
 * -1 automatic = the default: considered when this rank's share of the usable CPUs (affinity capped by the cgroup quota,
 * divided by LOCAL_WORLD_SIZE) is >= 6, no other local rank's GPU hangs off the same NUMA node and the batch has >= 4
 * chunks; the library then MEASURES: one call plain, one packed, afterwards whichever is clearly faster, the other re-probed every 32nd call
 * (packing gains ~16 % with one GPU per socket and loses with four). SR_PACK12=0|1 overrides the automatic choice,
 * SR_PACK_THREADS the worker count (default: CPU share - 3, at most 10). */
int sr_set_transport(sr_handle *h, int mode);
/* transport statistics of the last sr_recognise_batch call: chunks sent packed / plain, bytes copied host -> device */
int sr_transport_stats(const sr_handle *h, uint32_t *packed_chunks, uint32_t *plain_chunks, uint64_t *h2d_bytes);
/* test hooks: the host packer alone (variant 0 scalar, 1 AVX2, 2 AVX-512 VBMI, 3 AVX-512 VBMI with non-temporal stores, -1 best available, 100+N the N-thread worker pool; returns the OR
 * of all samples or 0xFFFFFFFF if the variant is unavailable; no GPU needed) and the device expander alone */
uint32_t sr_debug_pack12_host(int variant, const uint16_t *src, uint64_t n, uint8_t *dst);
int sr_debug_unpack12(sr_handle *h, const uint8_t *packed, uint64_t n, uint16_t *out);

/* Per-kernel device timing: after sr_timing_enable(h, max_records) every launch of the recognition-path kernels
 * by this handle's noise_atap, VAD, MFCC, DTW, recognise, enrol, path and averaging calls (host-buffer and _dev forms) is bracketed
 * by a CUDA event pair on the launching stream. Not timed: the test-hook kernels (FFT, get_dis, get_mdl, dtw_limit,
 * sqrt check), the packed transport's 12-bit expander, the slot packing of enrol and averaging and the streaming pool's kernels. Zero-size
 * calls launch and record nothing. sr_timing_collect synchronises the
 * stream and returns (tag, milliseconds) per timed launch in issue order, then rearms. Tags: 0 noise_atap+VAD,
 * 1 get_mfcc, 2 status, 3 best-init, 4 dtw (greedy), 5 best-final, 6 dtw (banded DP, in sr_dtw_batch* and in recognise
 * calls under the SR_DTW_BAND matcher), 7 the banded DP with its path (every pass of sr_dtw_path_batch and
 * sr_average_bank that aligns), 8 sr_average_bank's template update, 9 the connected-word decoder (sr_connected_batch,
 * sr_recognise_connected_batch; their get_mfcc launches are tag 1), 10 the grammar decoder (sr_connected_grammar_batch,
 * sr_recognise_connected_grammar_batch; their get_mfcc launches are tag 1), 11 and 12 the long-form block and segment passes
 * (include/sr_long.h), 14 dtw (the symmetric P = 1 DP, in sr_dtw_batch* and in recognise calls under the SR_DTW_SYM_P1
 * matcher), 15 the resampling of a staged group to 8 kHz (the long-form calls at a rate of include/sr_synth.h), of a
 * chunk (sr_recognise_batch_at_rate) or of a whole batch (the other capture calls at a rate of include/sr_synth.h).
 * max_records = 0 disables. */
int sr_timing_enable(sr_handle *h, uint32_t max_records);
int sr_timing_collect(sr_handle *h, uint32_t *tags, float *ms, uint32_t cap, uint32_t *n);

/* Kernel variant of the greedy dtw (both bit-identical): 0 = one lane per (utterance, template) pair for the whole walk,
 * 1 = pairs handed to lanes dynamically from a ring of staged utterances (no lane waits for the longest walk of its
 * warp), -1 = the library default (SR_DTW_VARIANT=0|1 overrides it). */
int sr_set_dtw_variant(sr_handle *h, int variant);

/* number of kernel launches this handle has issued (bench.py reports it as gpu_launches) */
uint64_t sr_launch_count(const sr_handle *h);

#ifdef __cplusplus
}
#endif
#endif /* SPEECH_RECOG_H_ */
