// sr_internal.h -- private to the library: the handle, workspaces and launch prototypes shared by sr_api.cu
// and sr_stream.cu. Nothing here is part of the C-ABI.
#pragma once
#include <chrono>
#include <deque>
#include <functional>
#include <memory>
#include <mutex>
#include <new>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <string>
#include <thread>
#include <vector>
#include "sr_dtw_core.cuh"
#include "sr_resample_core.cuh"
#include "../../include/sr_long_grammar.h"

namespace srk {
cudaError_t launch_vad(const u16 *pcm, u32 U, u32 B, u32 n_len, u32 buf_len, int do_atap, int do_vad, atap_tag *atap,
                       u32 *seg_off, int num_sms, cudaStream_t st, u32 *work = nullptr);
cudaError_t launch_mfcc(const u16 *pcm, u32 U, u32 B, const u32 *seg, u32 seg_stride, const atap_tag *atap, void *ftr,
                        int num_sms, cudaStream_t st, const u32 *row_map = nullptr, u32 rows_total = 0,
                        const u32 *B_dev = nullptr, u32 *work = nullptr);
cudaError_t launch_mfcc_geomb(const u16 *pcm, u32 U, u32 B, const u32 *seg, u32 seg_stride, const atap_tag *atap, void *ftr,
                              int num_sms, cudaStream_t st, const u32 *row_map = nullptr, const u32 *B_dev = nullptr);
cudaError_t launch_fft_generic(const u32 *in_packed, const s16 *frames, u32 len, u32 n, u32 *raw_out, u32 *mag,
                               cudaStream_t st);
cudaError_t launch_fft_raw_n(const u32 *in, u32 N, u32 n, u32 *out, cudaStream_t st);
cudaError_t launch_log100_check(u64 lo, u64 hi, unsigned long long *bad_dev, cudaStream_t st);
cudaError_t launch_mag10_check(int which, u64 lo, u64 hi, unsigned long long *bad_dev, cudaStream_t st);
// n keys (B argmin keys, or a decision rule's B * C keys) set to main.c:276-278's start
cudaError_t launch_best_init(u64 *best, u64 n, cudaStream_t st);
// The decision of B inputs into the fields (sr_dtw.cu): without a rule (rl.C = 0) from the argmin keys keys = best;
// under one from the keys [B][rl.C], with the decision's keys into best[B] and SR_ST_REJECT into status
cudaError_t launch_best_final(u64 *best, const u64 *keys, u32 B, const Rule &rl, u32 *best_idx, u32 *best_dis, u32 *cmd,
                              u8 *status, cudaStream_t st);
cudaError_t launch_status(const u32 *seg_off, const void *ftr, u32 B, u8 *status, cudaStream_t st);
cudaError_t launch_get_dis(const s16 *a, const s16 *b, u32 n, u32 *out, cudaStream_t st);
cudaError_t launch_dtw_limit(const u16 *x, const u16 *y, const u16 *I, const u16 *M, u32 n, u8 *out, cudaStream_t st);
cudaError_t launch_get_mdl(const void *in1, const void *in2, void *mdl, u32 n, u32 *dis, cudaStream_t st);
cudaError_t launch_pack_slots(const void *ftr, const u8 *status, u32 B, void *bank, u32 slot_stride, cudaStream_t st);
// the banded DP with its warping path over a list of (input, template, output) u32 triples (NULL: p, p, p), and the DBA
// update of G groups of K bank slots (sr_dtw_align.cu)
cudaError_t launch_dtw_align(const void *in_base, u32 in_stride, const void *tpl_base, u32 tpl_stride, const void *pairs,
                             u32 n, int band_r, u8 *path, u32 *path_len, u32 *dis, const u32 *pick_S, const u32 *mask, u32 K,
                             void *tpl_out, u32 *anchor_out, int num_sms, cudaStream_t st);
cudaError_t launch_average_update(const void *bank, u32 slot_stride, u32 K, u32 G, const u32 *mask, const u8 *path,
                                  const u32 *path_len, void *tpl, cudaStream_t st);
// the connected-word decoder over sequences [b0, b0 + nb) of a batch, nb <= kSeqChunk (seq_off: [B][2] first row, first
// word record, or NULL: b * frm_stride, b * max_words), the gather of get_mfcc pieces into long feature rows and the join
// of a capture's segments (sr_dtw_connected.cu)
cudaError_t launch_dtw_connected(const s16 *feat, u32 frm_stride, const u32 *frm_num, const u32 *seq_off, u32 b0, u32 nb,
                                 const void *bank, u32 T, u32 slot_stride, u32 penalty, u32 max_words, sr_conn_word *words,
                                 u32 *n_words, u64 *total, cudaStream_t st);
cudaError_t launch_conn_gather(const void *pf, const u32 *pdst, u32 P, s16 *feat, int num_sms, cudaStream_t st);
cudaError_t launch_conn_concat(const u32 *seq_of, const u32 *seq_off, const sr_conn_word *seq_words, const u32 *seq_nw,
                               const u64 *seq_total, u32 B, u32 max_words, sr_conn_word *words, u32 *n_words, u64 *total,
                               cudaStream_t st);
// the grammar decoder over sequences [b0, b0 + nb) of a batch, nb <= kSeqChunk (seq: [B][3] first feature row, first
// record row, segment first frames) against C copies of bank slots (copy: [C] slot | state << 8 | src << 16), records in
// rec (sr_dtw_connected.cu)
cudaError_t launch_dtw_grammar(const s16 *feat, const u32 *frm_num, const u32 *seq, u32 b0, u32 nb, const void *bank, u32 slot_stride,
                               const u32 *copy, u32 C, u32 S, u32 final_mask, u32 penalty, u32 max_words, sr_conn_word *words,
                               u32 *n_words, u64 *total, u64 *rec, cudaStream_t st);
// the long-recording grammar decoder over sequences [b0, b0 + nb) (seq: [B][4] first segment, segments, frames, first
// record row) of a flat segment table (seg_row: first feature row, seg_frm: frames), records in recD / recS
// (sr_dtw_connected.cu)
cudaError_t launch_dtw_long_grammar(const s16 *feat, const u32 *seq, u32 b0, u32 nb, const u32 *seg_row, const u32 *seg_frm,
                                    const void *bank, u32 slot_stride, const u32 *copy, u32 C, u32 S, u32 final_mask, u32 penalty,
                                    u32 max_words, sr_conn_word *words, u32 *n_words, u64 *total, u64 *recD, u32 *recS,
                                    cudaStream_t st);
cudaError_t launch_sqrt_check(u32 lo, u32 hi, unsigned long long *bad_dev, cudaStream_t st);
cudaError_t launch_unpack12(const void *packed, u64 n_samples, u16 *out, cudaStream_t st);
// the long-form VAD and its per-segment recognition (sr_vad_long.cu): noise_atap, the block summaries into info
// ([B][long_info_stride(U)] words), the segment pass, the flat segment table (step 0: the prefix sum into first / n_flat,
// step 1: the table), the per-segment status and the scatter of the argmin into the records
u32 long_info_stride(u32 U);
cudaError_t launch_long_atap(const u16 *pcm, u32 U, u32 B, const u32 *lens, u32 n_len, atap_tag *atap, cudaStream_t st);
cudaError_t launch_long_blocks(const u16 *pcm, u32 U, u32 B, const u32 *lens, const atap_tag *atap, u32 *info, int num_sms,
                               cudaStream_t st);
cudaError_t launch_long_segments(u32 U, u32 B, const u32 *lens, const atap_tag *atap, const u32 *info, u32 max_segs, u32 *n_segs,
                                 u32 *seg_off, cudaStream_t st);
cudaError_t launch_long_flatten(const u32 *n_segs, const u32 *seg_off, const atap_tag *atap, u32 B, u32 max_segs, u32 *first,
                                u32 *n_flat, u32 *seg2, u32 *row, u32 *slot, atap_tag *atap_seg, cudaStream_t st, int step);
cudaError_t launch_long_status(const u32 *seg2, const void *ftr, const u32 *n_flat, u32 M, u8 *status, cudaStream_t st);
cudaError_t launch_long_scatter(const u32 *seg2, const u32 *slot, const void *ftr, const u8 *status, const u64 *best,
                                const u32 *n_flat, u32 M, sr_long_seg *rec, const Rule &rl, cudaStream_t st);
class PackPool;
}  // namespace srk

using namespace srk;

inline thread_local std::string g_tls_error;

struct sr_comm;                                       // sr_comm.cu: NCCL communicator + its stream
struct sr_handle;

// grow-only device buffer (ensure), freed with its owner: owners are deleted under a DeviceGuard of their device
struct DevBuf {
    void *p = nullptr;
    size_t cap = 0;
    DevBuf() = default;
    DevBuf(const DevBuf &) = delete;
    DevBuf &operator=(const DevBuf &) = delete;
    ~DevBuf() { if (p) cudaFree(p); }
};

// pinned host buffer, freed with its owner
template <class T> struct Pinned {
    T *p = nullptr;
    Pinned() = default;
    Pinned(const Pinned &) = delete;
    Pinned &operator=(const Pinned &) = delete;
    ~Pinned() { reset(); }
    void reset() { if (p) cudaFreeHost(p); p = nullptr; }
    cudaError_t alloc(size_t bytes) {
        reset();
        const cudaError_t e = cudaMallocHost(reinterpret_cast<void **>(&p), bytes);
        if (e != cudaSuccess) p = nullptr;
        return e;
    }
};

// The packed PCM transport of sr_recognise_batch (sr_transport.cu). Chunks whose samples are all < 4096 cross PCIe as
// 12 bits per sample: a worker pool packs them from the back of the batch into pinned staging slots while the caller's
// thread sends plain u16 chunks from the front. Owns the pool, the pinned and device staging, the automatic mode's
// measurements and the statistics of the last call.
class PackedTransport {
public:
    // sends chunk c into device PCM buffer buf (0 or 1): from packed_src (12-bit, pinned staging) or, if NULL, plain
    using Step = std::function<int(uint32_t c, int buf, const void *packed_src)>;
    int mode = -1;                                      // sr_set_transport: 0 off, 1 on, -1 automatic
    uint32_t last_packed = 0, last_plain = 0;           // sr_transport_stats: chunks and bytes of the last call
    uint64_t last_h2d = 0;
    ~PackedTransport();
    // every chunk of `chunk` utterances (the last one shorter) of pcm[B][U], once, through step
    int send(sr_handle *h, const uint16_t *pcm, uint32_t U, uint32_t B, uint32_t chunk, const Step &step);
    // call after the results of the call are on the host: the automatic mode times the whole call
    void call_done(uint64_t pcm_bytes);
    // device staging of buffer buf, where step copies a packed chunk to
    unsigned char *device_stage(int buf) const { return static_cast<unsigned char *>(dpacked.p) + (size_t)buf * stage_cap; }

private:
    static constexpr int kStage = 4;
    uint64_t auto_calls = 0;                            // automatic mode: calls seen, measured ns per PCM byte [plain, packed]
    double auto_ns_per_byte[2] = {0.0, 0.0};
    bool probe = false;                                 // the current call is a measurement of the automatic mode
    std::chrono::steady_clock::time_point t_call0;
    std::unique_ptr<PackPool> pool;
    Pinned<uint8_t> stage[kStage];
    size_t stage_cap = 0;
    DevBuf dpacked;                                     // 2 x stage_cap
    int resolved_mode(const sr_handle *h) const;
    bool auto_pick();
    bool setup(const sr_handle *h, size_t pk);
    int send_packed(sr_handle *h, const uint16_t *pcm, uint32_t U, uint32_t B, uint32_t chunk, const Step &step);
};

// a template bank on the device: n flash-layout slots of `stride` bytes at p, walked in `order` (NULL: slot order)
struct BankView {
    const void *p = nullptr;
    u32 n = 0, stride = 0;
    const u32 *order = nullptr;
};

struct sr_handle {
    int device = 0;
    int num_sms = 132;
    cudaStream_t own_stream = nullptr;
    cudaStream_t stream = nullptr;
    cudaStream_t copy_stream = nullptr;                 // H2D of the next chunk while the current one computes
    cudaEvent_t ev_h2d[2] = {nullptr, nullptr}, ev_done[2] = {nullptr, nullptr};
    uint64_t launches = 0;
    std::string err;
    // template bank (sr_set_bank*). Its order lists the slots in ascending frm_num order (only for banks wider than one
    // 32-template tile): a hint for the greedy dtw kernels, recomputed when the bank pointer / geometry changes;
    // correctness never depends on it
    BankView bank;
    DevBuf bank_own, bank_perm;
    const void *perm_bank = nullptr;
    u32 perm_n = 0, perm_stride = 0;
    // optional per-kernel timing (sr_timing_enable): event pairs recorded around every launch
    bool timing = false;
    std::vector<cudaEvent_t> ev;
    std::vector<uint32_t> ev_tag;
    size_t ev_used = 0;
    PackedTransport transport;                          // of sr_recognise_batch
    // command labels (commstr, main.c:25-31): n_labels records of label_stride bytes, NUL-terminated
    std::vector<uint8_t> labels;
    u32 n_labels = 0, label_stride = 0;
    sr_comm *comm = nullptr;                           // the exchange step (sr_comm_create), optional
    int dtw_variant = -1;                              // greedy dtw kernel: 0 static lane = pair (sr_dtw.cu), 1 dynamic pairs (sr_dtw_dyn.cuh), -1 default
    u32 match_flags = 0;                               // matcher of the recognition calls (sr_set_match): 0 greedy walk, SR_DTW_BAND (| SR_DTW_ANY_RATE) or SR_DTW_SYM_P1,
                                                       // | SR_DTW_LIFTER | SR_DTW_KNN(k) | SR_DTW_REJECT(q)
    int match_r = 0;                                   // its band radius
    DevBuf mfcc_work;                                  // the same for mfcc_kernel (next utterance, CTAs finished)
    DevBuf vad_work;                                   // two words: dynamic utterance hand-out of vad_kernel (zeroed once, self re-arming)
    DevBuf dtw_scratch;                                // one word: max frm_num of the current inputs (dynamic kernel's slot size)
    int geom = 0;                                      // SR_GEOM_REF (160/80/1024) or SR_GEOM_B (200/80/256, extension)
    int numa_node = -1;                                // node the device hangs off (-1 unknown / single node)
    // grow-only device workspaces; scratch[] serves the secondary entry points (FFT, get_dis, get_mdl, dtw_limit, the
    // 12-bit expander, the sqrt check, enrol's bank image, dtw()'s one-slot bank) and is never read by a recognise call
    DevBuf pcm, atap, seg, ftr, score, best, best_alt, status, bidx, bdis, cmd, scratch[3];
    // pcm8: input staged in pcm at another rate, resampled to 8 kHz by K15 for the 8 kHz body to read. The capture calls
    // at a rate: sr_recognise_batch_at_rate (one chunk, [nb][U8]), sr_enrol_batch_at_rate,
    // sr_recognise_connected_batch_at_rate, sr_recognise_connected_grammar_batch_at_rate (the whole batch, [B][U8]);
    // the long-form calls at a rate: sr_recognise_long_batch_at_rate, sr_recognise_long_grammar_batch_at_rate (one
    // staged group, [G][U8])
    DevBuf pcm8;
    // The workspace table of the other call families: one buffer per thing held, each listed with what it holds and the
    // calls that use it. Where calls put different things in one buffer, each call's contents are named.
    //
    // get_mfcc pieces of long segments, at most kPieceChunk per launch (run_pieces): sr_mfcc_long_batch,
    // sr_recognise_connected_batch, sr_recognise_connected_grammar_batch, sr_recognise_long_grammar_batch
    // - seg, row, dst: [P][2] start / end sample, [P] PCM row, [P][2] first long feature row / frames
    // - atap, ftr: [P] the recording's atap, [P] the piece's features
    struct { DevBuf seg, row, dst, atap, ftr; } pieces;
    // connected words
    // - feat: long feature rows. sr_mfcc_long_batch, sr_connected_batch, sr_recognise_connected_batch,
    //   sr_connected_grammar_batch, sr_recognise_connected_grammar_batch, sr_connected_grammar_segs_batch,
    //   sr_recognise_long_grammar_batch
    // - seq_frm: frames per sequence. sr_connected_batch (the caller's frm_num), sr_recognise_connected_batch
    // - seq_off, seq_of: [n][2] each sequence's first row and first word record, [B][3] each capture segment's sequence.
    //   sr_recognise_connected_batch
    // - seq_words, seq_total, seq_n_words: each sequence's word records, total and word count. sr_recognise_connected_batch
    // - words, n_words, total: the caller's outputs (conn_outputs). sr_connected_batch, sr_recognise_connected_batch,
    //   sr_connected_grammar_batch, sr_recognise_connected_grammar_batch, sr_connected_grammar_segs_batch,
    //   sr_recognise_long_grammar_batch
    struct { DevBuf feat, seq_frm, seq_off, seq_of, seq_words, seq_total, seq_n_words, words, n_words, total; } conn;
    // both grammar decoders: run_grammar (sr_connected_grammar_batch, sr_recognise_connected_grammar_batch) and K13's
    // run_long_grammar (sr_connected_grammar_segs_batch, sr_recognise_long_grammar_batch)
    // - seq: the sequence table. run_grammar: [B][3]; K13: [B][4]
    // - frm: run_grammar: frames per sequence; K13: frames per segment
    // - seg_row: each segment's first feature row. K13
    // - rec: records. run_grammar's; K13's 64-bit ones
    // - rec_state: K13's 32-bit records
    // - copy: the copy table (stage_copies). Both decoders
    // - vad_segs: a group's long-form VAD segments. sr_recognise_long_grammar_batch
    struct { DevBuf seq, frm, seg_row, rec, rec_state, copy, vad_segs; } gram;
    // long-form VAD and recognition (sr_long.h)
    // - info: block summaries (vad_long_impl). sr_vad_long_batch(_dev), sr_recognise_long_batch(_dev),
    //   sr_recognise_long_grammar_batch
    // - seg_off: the segments [B][max_segs][2]. sr_recognise_long_batch(_dev)
    // - first, n_flat, seg2, row, slot, atap_seg, status, keys, ftr: the flat segment table (recognise_segs_impl): [B]
    //   each recording's first flat segment, their count, [M][2] start / end sample, [M] PCM row, [M] record slot,
    //   [M] atap, status, argmin or decision-rule keys, features. sr_recognise_long_batch(_dev)
    // - atap, n_segs: [B] atap records and segment counts. sr_recognise_long_batch_dev (when the caller passes none),
    //   sr_vad_long_batch, sr_recognise_long_batch, sr_recognise_long_grammar_batch
    // - per_seg: the caller's per-segment output. sr_vad_long_batch: seg_off; sr_recognise_long_batch: the records
    // - lens: the caller's lens. sr_vad_long_batch, sr_recognise_long_batch, sr_recognise_long_grammar_batch and their
    //   _at_rate forms (there in input samples)
    // - lens8: every recording's 8 kHz length [B] (its samples are in pcm8). sr_recognise_long_batch_at_rate,
    //   sr_recognise_long_grammar_batch_at_rate
    struct { DevBuf info, seg_off, first, n_flat, seg2, row, slot, atap_seg, status, keys, ftr, atap, n_segs, per_seg, lens, lens8; } lng;
    // alignment: sr_dtw_path_batch and sr_average_bank
    // - in_bank: sr_dtw_path_batch: in; sr_average_bank: the bank image
    // - mdl_out: sr_dtw_path_batch: mdl; sr_average_bank: the output bank image
    // - path: the warping paths. Both
    // - len_pairs: sr_dtw_path_batch: path_len; sr_average_bank: the pair list
    // - dis_tpl: sr_dtw_path_batch: dis; sr_average_bank: the group templates
    // - mask, group_status, anchor_S, slot_len: [G] member masks, [G] group status, [slots][K] anchor scores, [slots] path
    //   lengths. sr_average_bank
    struct { DevBuf in_bank, mdl_out, path, len_pairs, dis_tpl, mask, group_status, anchor_S, slot_len; } align;
    int best_sel = 0;                                  // which of best / best_alt the current recognise call uses (alternates when a
                                                       // communicator is attached: the previous call's keys may still be being gathered)
};

// the key buffer of the current recognise call
inline DevBuf &key_buf(sr_handle *h) { return h->best_sel ? h->best_alt : h->best; }

inline int fail(sr_handle *h, const char *what, cudaError_t e) {
    char buf[512];
    snprintf(buf, sizeof buf, "%s: %s", what, e == cudaSuccess ? "invalid argument" : cudaGetErrorString(e));
    g_tls_error = buf;
    if (h) h->err = buf;
    return e == cudaSuccess ? -1 : (int)e;
}
#define SR_CK(h, call)                                           \
    do {                                                         \
        cudaError_t e__ = (call);                                \
        if (e__ != cudaSuccess) return fail((h), #call, e__);    \
    } while (0)
#define SR_REQUIRE(h, cond)                                      \
    do {                                                         \
        if (!(cond)) return fail((h), "requirement failed: " #cond, cudaSuccess); \
    } while (0)

// ---- kernel launches: every one is counted (sr_launch_count); the tagged ones are timed ----------------------------
enum { TAG_NONE = -1, TAG_VAD = 0, TAG_MFCC = 1, TAG_STATUS = 2, TAG_BEST_INIT = 3, TAG_DTW = 4, TAG_BEST_FINAL = 5,
       TAG_DTW_BAND = 6, TAG_ALIGN = 7, TAG_AVG_UPDATE = 8, TAG_CONN = 9,
       TAG_GRAM = 10, TAG_LONG_BLOCKS = 11, TAG_LONG_SEGS = 12, TAG_LONG_GRAM = 13, TAG_DTW_SYM = 14, TAG_RESAMPLE = 15 };

// one kernel launch on the handle's stream, launch() returning its cudaError_t (for <<<a, b>>>: cudaGetLastError()):
// bracketed by an event pair when tag is not TAG_NONE and timing is enabled, counted when it succeeds
template <class F> inline int launch_on(sr_handle *h, int tag, const char *what, F launch) {
    size_t slot = SIZE_MAX;
    if (tag != TAG_NONE && h->timing && (h->ev_used + 1) * 2 <= h->ev.size()) {
        slot = h->ev_used++;
        h->ev_tag[slot] = tag;
        cudaEventRecord(h->ev[2 * slot], h->stream);
    }
    const cudaError_t e = launch();
    if (slot != SIZE_MAX) cudaEventRecord(h->ev[2 * slot + 1], h->stream);
    if (e != cudaSuccess) return fail(h, what, e);
    ++h->launches;
    return 0;
}
#define SR_LAUNCH(h, tag, call)                                                                   \
    do {                                                                                          \
        if (const int rc__ = launch_on((h), (tag), #call, [&] { return (call); })) return rc__;   \
    } while (0)

// samples per frame in the handle's geometry
inline u32 frame_len(const sr_handle *h) { return h->geom == SR_GEOM_B ? 200u : SR_FRAME_LEN; }

inline cudaError_t ensure(DevBuf &b, size_t bytes) {
    if (bytes <= b.cap) return cudaSuccess;
    if (b.p) { cudaError_t e = cudaFree(b.p); b.p = nullptr; b.cap = 0; if (e != cudaSuccess) return e; }
    size_t want = bytes + (bytes >> 3) + 256;
    cudaError_t e = cudaMalloc(&b.p, want);
    if (e != cudaSuccess) { b.p = nullptr; return e; }
    b.cap = want;
    return cudaSuccess;
}
// ensure, with p set to the workspace
template <class T> inline cudaError_t ensure(DevBuf &b, size_t bytes, T *&p) {
    const cudaError_t e = ensure(b, bytes);
    p = static_cast<T *>(b.p);
    return e;
}
// the caller's buffer p, or when it is NULL workspace b grown to `bytes`
template <class T> inline cudaError_t caller_or_ws(DevBuf &b, size_t bytes, T *&p) { return p ? cudaSuccess : ensure(b, bytes, p); }

inline u32 *mfcc_work(sr_handle *h) {
    if (!h->mfcc_work.p) {
        if (ensure(h->mfcc_work, 16) != cudaSuccess) { cudaGetLastError(); return nullptr; }
        if (cudaMemsetAsync(h->mfcc_work.p, 0, 16, h->stream) != cudaSuccess) { cudaGetLastError(); return nullptr; }
    }
    return static_cast<u32 *>(h->mfcc_work.p);
}

// get_mfcc in the handle's geometry
inline cudaError_t launch_mfcc_h(sr_handle *h, const u16 *pcm, u32 U, u32 B, const u32 *seg, u32 seg_stride, const atap_tag *atap,
                                 void *ftr, const u32 *row_map = nullptr, u32 rows_total = 0, const u32 *B_dev = nullptr) {
    if (h->geom == 1) return launch_mfcc_geomb(pcm, U, B, seg, seg_stride, atap, ftr, h->num_sms, h->stream, row_map, B_dev);
    return launch_mfcc(pcm, U, B, seg, seg_stride, atap, ftr, h->num_sms, h->stream, row_map, rows_total, B_dev, mfcc_work(h));
}

// the handle's work counters for vad_kernel (allocated and zeroed on first use)
inline u32 *vad_work(sr_handle *h) {
    if (!h->vad_work.p) {
        if (ensure(h->vad_work, 16) != cudaSuccess) { cudaGetLastError(); return nullptr; }
        if (cudaMemsetAsync(h->vad_work.p, 0, 16, h->stream) != cudaSuccess) { cudaGetLastError(); return nullptr; }
    }
    return static_cast<u32 *>(h->vad_work.p);
}

// The template scan's matcher, decoded once from the matcher flags and band radius (scan_plan): the matcher, the
// kernels' check_sign, guard (the 2:1 length guard, off under SR_DTW_ANY_RATE) and lifter, the radius clamped to 118,
// the timing tag (TAG_DTW, TAG_DTW_BAND or TAG_DTW_SYM) and the decision rule
struct ScanPlan {
    enum Matcher { kGreedy, kBand, kSym } matcher;
    bool check_sign, guard, lift;
    int r, tag;
    Rule rule;
};
// The plan of a scan against T templates under flags and band_r, false for flags the library refuses. rules: the
// recognition calls, whose flags are SR_DTW_CHECK_SIGN | sr_set_match's (any radius >= 0; a decision rule's C from T,
// none when T is 0); else sr_dtw_batch*, which have no status to decide a rule into (no bit >= 16, bits 4-15 other
// than SR_DTW_LIFTER ignored, a DP's radius >= 0 when T > 0, rule {0, 0, 0}).
bool scan_plan(u32 flags, int band_r, u32 T, bool rules, ScanPlan *out);
// the arguments of the scan of B inputs at in_ftr against bank under p (score, best, status and B_dev may be NULL)
ScanArgs scan_args(const ScanPlan &p, const BankView &bank, const void *in_ftr, u32 B, u32 *score, u64 *best,
                   const u8 *status, const u32 *B_dev = nullptr);
// The template scan under p (sr_dtw.cu) -- the one place a matcher becomes a kernel launch: the greedy walk with the
// handle's variant (sr_set_dtw_variant, else SR_DTW_VARIANT: 0 the static kernel, 1 the dynamic pairs), the banded DP
// (the thread form at r = 10, the warp-scan form for the other r <= 15, the whole-row form for r >= 16) or the symmetric
// DP, each in its liftered form under SR_DTW_LIFTER. One counted launch, also for the dynamic kernel's pre-pass.
cudaError_t launch_scan(sr_handle *h, const ScanPlan &p, const ScanArgs &a);

// the two handles' recognition calls score and decide alike: both greedy, or both the same DP (SR_DTW_ANY_RATE included)
// at the same radius, with or without SR_DTW_LIFTER alike, under the same decision rules
inline bool same_match(const sr_handle *a, const sr_handle *b) {
    ScanPlan p;
    scan_plan(a->match_flags, a->match_r, 0, true, &p);               // flags and radius sr_set_match accepted
    return a->match_flags == b->match_flags && (p.matcher == ScanPlan::kGreedy || a->match_r == b->match_r);
}

int comm_wait_before_scan(sr_handle *h, const void *score);   // sr_comm.cu
int recognise_dev_impl(sr_handle *h, const uint16_t *pcm, uint32_t U, uint32_t B, uint32_t n_len, const sr_recog_out *o,
                       bool wait_comm);             // sr_api.cu

struct DeviceGuard {
    int prev = -1;
    bool ok = true;
    explicit DeviceGuard(int dev) {
        if (cudaGetDevice(&prev) != cudaSuccess) { ok = false; return; }
        if (prev != dev && cudaSetDevice(dev) != cudaSuccess) ok = false;
    }
    ~DeviceGuard() { if (prev >= 0) cudaSetDevice(prev); }
};


#define D2H(h, dst, src, bytes) SR_CK(h, cudaMemcpyAsync((dst), (src), (bytes), cudaMemcpyDeviceToHost, (h)->stream))

// ---- the part every streaming pool shares (sr_stream.cu): K4's fixed captures and K14's live streams ----------------
// A push's step kernel appends the chunk and lists the segments it closed in ev / seg_ev / atap_ev / map_ev (n_ev of them,
// at most cap); stream_core_recognise then runs get_mfcc on seg_ev (offsets inside PCM row map_ev of a [S][row_len]
// buffer), the status, the handle's matcher and the packing of one sr_stream_event per segment, copies them back with the
// push's one synchronisation and hands them out behind any queued ones. The step kernels list them through
// srk::StreamEvents (sr_vad_core.cuh).
struct StreamCore {
    sr_handle *h = nullptr;
    u32 S = 0, cap = 0, stage_stride = 0;
    DevBuf stage, lens, ev, seg_ev, atap_ev, map_ev, n_ev, ftr, status, frm, out;
    Pinned<unsigned char> out_host;                // [count u32, pad][records]
    Pinned<u32> lens_host;                         // staging of a ragged push's lengths
    std::deque<sr_stream_event> pending;           // events not yet handed to the caller (max_events too small)
    static constexpr u32 kQuick = 4096;            // records fetched with the count in the first D2H copy
};
// the per-push buffers for S streams and cap events
cudaError_t stream_core_alloc(StreamCore &c, sr_handle *h, u32 S, u32 cap);
// a ragged push's lengths into lens_host (lens NULL: uniform_len for every stream); returns the longest
u32 stream_core_lens(StreamCore &c, const uint32_t *lens, u32 uniform_len);
// the chunk as the step kernel reads it (pinned host memory in place, else a staging copy), the lengths (ragged) and
// the event counter zeroed, on the handle's stream
int stream_core_stage(StreamCore &c, const uint16_t *chunk, u32 chunk_stride, u32 max_len, bool ragged, const u16 **chunk_dev,
                      u32 *chunk_dev_stride);
int stream_core_recognise(StreamCore &c, const u16 *pcm, u32 row_len, sr_stream_event *events, u32 max_events, u32 *n_events);
void stream_core_fetch(StreamCore &c, sr_stream_event *events, u32 max_events, u32 *n_events);

// ---- a streaming pool's input at a rate other than 8 kHz (sr_stream.cu), for K4 and K14 alike ------------------------
// Each push runs stream_resample_kernel before the pool's step kernel: it turns every stream's chunk into the 8 kHz
// outputs whose filter support has arrived (resample_ready, sr_resample_core.cuh) and carries the stream's input count
// and last K - 1 inputs to the next push. The step kernel reads the outputs through its ragged path. At 8 kHz there is
// no stage (hp == NULL) and the pool is the plain one.
struct ResampleStage {
    ResampleRate rate{8000, 1, 1, 1, 0};
    const int32_t *hp = nullptr;                   // the rate's [L][K] phase table on the pool's device
    u32 T = 0, out_stride = 0, hist_stride = 0, grid = 0;   // outputs per window, row strides, launch width
    size_t smem = 0;
    DevBuf out, lens, n, hist;                     // 8 kHz staging [S][out_stride] and its counts [S]; input counts [S]
                                                   // and carried inputs [S][hist_stride]
};
// the stage of S streams at `rate` whose pushes hold at most max_in input samples (nothing at 8 kHz); sets the kernel's
// dynamic shared-memory limit to what the largest rate needs, the same value whichever pool sets it
cudaError_t resample_stage_alloc(ResampleStage &r, sr_handle *h, u32 S, u32 rate, u32 max_in);
// one launch on the handle's stream: the chunk (*chunk, *stride; *lens, or *uniform_len when NULL) becomes each stream's
// new 8 kHz outputs below index `keep`, and *chunk .. *uniform_len then describe those outputs. Nothing at 8 kHz.
int resample_stage_push(ResampleStage &r, sr_handle *h, u32 S, u32 keep, const u16 **chunk, u32 *stride, const u32 **lens,
                        u32 *uniform_len);
// in a reset kernel: stream s back to no input received, its carried inputs mid-code (no-op without a stage: n NULL)
__device__ __forceinline__ void resample_stage_restart(u32 s, u32 *n, int16_t *hist, u32 hist_stride) {
    if (!n) return;
    n[s] = 0;
    for (u32 i = 0; i < hist_stride; ++i) hist[(size_t)s * hist_stride + i] = 0;
}
