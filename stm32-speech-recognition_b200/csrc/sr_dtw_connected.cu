// sr_dtw_connected.cu -- K6: connected words by one-pass DP over the template bank (one-stage DTW, Ney 1984), and K6g:
// the same decoder under a finite-state grammar, over a network of template copies (EXTENSION: the reference decodes one
// word per VAD segment; both are checked against this project's own CPU restatements and plain Python references, parity
// unpinned).
//
// dtw_connected_kernel: one thread-block CLUSTER per feature sequence, one WARP per bank slot (kConnWarps slots per CTA,
// up to kConnCluster CTAs per cluster). A warp holds its template's rows in registers, lane l owning columns 4l .. 4l+3
// as in dtw_wide_kernel / dtw_align_kernel, and advances one input frame per step: one dp_column step (sr_dtw_core.cuh,
// which also gives the headroom of the keys) writes the template's column of D for that frame. Cells are 64-bit keys
//   key = D << 10 | (1023 - start)        (start = the input frame the cell's word started at, < 1024)
// so one unsigned min compares (D, -start) lexicographically: the smallest D, ties to the later start. Cell j = 0 also
// takes E(i-1) + penalty, a new word starting at frame i. After each frame every warp sends its end cell, re-keyed as
//   ekey = D << 17 | slot << 10 | start    (smallest D, ties to the lowest slot)
// to every CTA of the cluster through distributed shared memory (lane r stores to CTA r), one cluster barrier follows, and
// every warp reduces the candidates to E(i) itself; rank 0 records ekey per frame (818 x 8 B), and after the last frame
// one lane traces the words back through those records. Candidates are double-buffered by frame parity, so one barrier
// per frame suffices: a CTA writes frame i+2's candidates only after every CTA has passed barrier i+1, i.e. has read
// frame i's.
//
// dtw_grammar_kernel is dtw_connected_kernel with the bank replaced by the grammar's COPIES: a copy c = (state s', member
// slot t) exists when some arc into s' carries cmd(t), and enters from src(c), the states with such an arc. The host
// numbers the copies state-major, then by slot, and hands the kernel one word per copy,
//   copy[c] = slot | state << 8 | src << 16.
// One warp per copy (ceil(C / kConnWarps) <= 16 CTAs), each frame's column and end-cell exchange exactly as in K6, the
// copy index in the slot field of the ekey. After the cluster barrier
//   - each warp reduces only the candidates whose copy's state is in its own src mask: min_{s in src} E_s(i) + P is the
//     coupling term of its cell j = 0 at frame i + 1 (the state of every copy is kept in a shared byte table);
//   - global warp g reduces E_s(i) for the states s = g (mod warps in the cluster) and stores it, as an ekey, to the
//     sequence's record rows in global memory: rec[(rec0 + i) * S + s].
// At the first frame of a later segment every within-word cell is reset to +inf, so no word crosses the pause, while E and
// with it the grammar state carry over. After the last frame one lane of rank 0 picks the final state and traces back
// through the records, writing each word with its segment and segment-relative frames.
//
// conn_gather_kernel copies the rows of get_mfcc pieces into their long feature rows; conn_concat_kernel joins the words
// of the segments of one capture (sr_recognise_connected_batch).
#include <cooperative_groups.h>
#include <utility>
#include "sr_dtw_core.cuh"

namespace cg = cooperative_groups;

namespace srk {

constexpr int kConnWarps = 8;                              // bank slots or copies per CTA
constexpr int kConnCluster = 16;                           // CTAs per cluster at most: 128 slots or copies
constexpr int kConnCand = kConnWarps * kConnCluster;       // candidates per frame buffer
constexpr u32 kConnFrm = SR_CONN_FRM_MAX;                  // 818
constexpr u32 kSeqNrm = kConnFrm * 24;                     // norm offset of the sequence's byte-plane slot
constexpr int kSeqBytes = kConnFrm * 28;                   // 22 904
constexpr int kConnSmem = kSeqBytes + kConnWarps * kSlotBytes + 2 * kConnCand * 8 + kConnFrm * 8;   // 58 184
constexpr int kGramSmem = kSeqBytes + kConnWarps * kSlotBytes + 2 * kConnCand * 8 + kConnCand;      // 51 768
constexpr u64 kKeyInf = 1ull << 62;
constexpr u64 kEkeyNone = ~0ull;
constexpr u32 kSegNone = 1023u;                            // segment field of a segment without frames
static_assert(kConnCand == SR_CONN_SLOT_MAX && kConnCand == SR_GRAM_COPY_MAX, "one warp per slot or copy");
static_assert(kConnFrm < kSegNone, "start frames and segment first frames are 10-bit fields");

__device__ __forceinline__ u64 umin64(u64 a, u64 b) { return a < b ? a : b; }
__device__ __forceinline__ u64 warp_min(u64 v) {
#pragma unroll
    for (int o = 16; o; o >>= 1) v = umin64(v, __shfl_xor_sync(0xFFFFFFFFu, v, o));
    return v;
}

// The start of both kernels: the sequence's N rows as byte planes (stage_planes reads row r at src + 4 + 24 r: src is a
// header-less row array shifted by 4), then member(M), which stages what
// else the kernel needs and returns the warp's bank slot with M = its frame count (left 0: the warp walks nothing); that
// template's planes, one cluster barrier (staging done, and every CTA of the cluster runs), then lane l's four template
// rows in b and a column of +inf in D. Returns M.
template <class Member>
__device__ __forceinline__ u32 conn_prologue(cg::cluster_group &cl, unsigned char *smem, const unsigned char *src, u32 N, PRow (&b)[4],
                                             u64 (&D)[4], Member member) {
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    unsigned char *tslot = smem + kSeqBytes + warp * kSlotBytes;
    stage_planes(smem, kSeqNrm, src, (int)N, threadIdx.x, blockDim.x);
    u32 M = 0;
    const unsigned char *slot = member(M);
    if (M) stage_planes(tslot, kNrm119, slot, (int)M, lane, 32);
    cl.sync();
    const int j0 = lane * 4;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        if (M) load_row(b[k], tslot, kNrm119, j0 + k < (int)M ? j0 + k : 0);
        D[k] = kKeyInf;
    }
    return M;
}

// The column of input row a for a warp whose template has M >= 1 frames: one dp_column step on keys
// D << 10 | (1023 - start) with +inf = kInf, cell j = 0 entered from `enter`. Returns the end cell's key (>= kInf:
// unreached). The caller loads a: loaded in here, K6g's segment reset compiles to other code.
template <u64 kInf>
__device__ __forceinline__ u64 conn_column(const PRow &a, u32 M, u64 enter, const PRow (&b)[4], u64 (&D)[4]) {
    const int lane = threadIdx.x & 31, j0 = lane * 4;
    dp_column<u64, kInf>(D, lane, [&](int k, u64 up, u64 dg, u64 &d, u64 &A, bool &valid) {
        const int j = j0 + k;
        valid = j < (int)M;
        d = (u64)pdist(a, b[k]) << 10;
        A = umin64(up, j == 0 ? enter : dg);
    }, [](int, u64, u64) {});
    return dp_end(D, ((int)M - 1) & 3, ((int)M - 1) >> 2);
}

// Frame i of a warp whose template has M frames (0: none): its column by conn_column, then its end cell as
// ekey = D << 17 | idx << 10 | start to candidate idx of every CTA of the cluster, and one cluster barrier. Returns the
// frame's candidate buffer.
__device__ __forceinline__ u64 *conn_frame(cg::cluster_group &cl, u32 nc, const unsigned char *smem, u64 *cand, u32 i, u32 M,
                                           u64 enter, const PRow (&b)[4], u64 (&D)[4], u32 idx) {
    const int lane = threadIdx.x & 31;
    u64 mine = kEkeyNone;
    if (M) {
        PRow a;
        load_row(a, smem, kSeqNrm, (int)i);                // broadcast read
        const u64 e = conn_column<kKeyInf>(a, M, enter, b, D);
        if (e < kKeyInf) mine = ((e >> 10) << 17) | ((u64)idx << 10) | (u64)(1023u - (u32)(e & 1023u));
    }
    u64 *buf = cand + (i & 1) * kConnCand;
    if ((u32)lane < nc) cl.map_shared_rank(buf, (unsigned)lane)[idx] = mine;
    cl.sync();
    return buf;
}

__global__ void __launch_bounds__(kConnWarps * 32, 2)
dtw_connected_kernel(const s16 *__restrict__ feat, u32 frm_stride, const u32 *__restrict__ frm_num,
                     const u32 *__restrict__ seq_off /* [.][2] first row, first word record; NULL: b * frm_stride, b * max_words */,
                     const unsigned char *__restrict__ bank, u32 T, u32 slot_stride, u32 penalty, u32 max_words,
                     sr_conn_word *__restrict__ words /* or NULL */, u32 *__restrict__ n_words, u64 *__restrict__ total /* or NULL */) {
    extern __shared__ __align__(128) unsigned char smem_raw[];
    cg::cluster_group cl = cg::this_cluster();
    const u32 nc = cl.num_blocks(), rank = cl.block_rank();
    const u32 s = blockIdx.x / nc;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    u64 *cand = reinterpret_cast<u64 *>(smem_raw + kSeqBytes + kConnWarps * kSlotBytes);   // [2][kConnCand]
    u64 *rec = cand + 2 * kConnCand;                                                       // [kConnFrm] E(i) as ekey
    const u32 N = frm_num[s];
    if (N == 0) {                                          // the whole cluster leaves: no barrier, no remote store
        if (rank == 0 && threadIdx.x == 0) {
            n_words[s] = 0;
            if (total) total[s] = 0;
        }
        return;
    }
    const size_t row0 = seq_off ? seq_off[2 * s] : (size_t)s * frm_stride;
    const u32 t = rank * kConnWarps + warp;                // this warp's bank slot
    PRow b[4];
    u64 D[4];
    const u32 M = conn_prologue(cl, smem_raw, reinterpret_cast<const unsigned char *>(feat + row0 * 12) - 4, N, b, D, [&](u32 &M) {
        const unsigned char *slot = bank + (size_t)t * slot_stride;
        if (t < T) {
            const u32 frm = decode_frm(*reinterpret_cast<const u32 *>(slot), true);
            if (frm != kNoWalk) M = frm;
        }
        return slot;
    });
    const u64 pen = penalty;
    u64 enter = (pen << 10) | 1023u;                       // E(-1) + penalty, a word starting at frame 0
    const u32 ncand = nc * kConnWarps;
    for (u32 i = 0; i < N; ++i) {
        const u64 *buf = conn_frame(cl, nc, smem_raw, cand, i, M, enter, b, D, t);
        u64 best = kEkeyNone;
        for (u32 q = lane; q < ncand; q += 32) best = umin64(best, buf[q]);
        best = warp_min(best);
        if (rank == 0 && threadIdx.x == 0) rec[i] = best;
        enter = best == kEkeyNone ? kKeyInf : ((((best >> 17) + pen) << 10) | (u64)(1023u - (i + 1)));
    }
    if (rank != 0 || threadIdx.x != 0) return;
    // trace-back through the per-frame records: the word ending at frame i is [start, i + 1) of slot, entered from E(start-1)
    const u64 last = rec[N - 1];
    if (last == kEkeyNone) {                               // no member in the bank
        n_words[s] = 0;
        if (total) total[s] = ~0ull;
        return;
    }
    u32 K = 0;
    for (int i = (int)N - 1; i >= 0; i = (int)(rec[i] & 1023u) - 1) ++K;
    const size_t w0 = seq_off ? seq_off[2 * s + 1] : (size_t)s * max_words;
    const u32 cap = seq_off ? N : max_words;
    u32 k = K;
    for (int i = (int)N - 1; i >= 0;) {
        const u64 r = rec[i];
        const u32 st = (u32)(r & 1023u), slot = (u32)((r >> 10) & 127u);
        const u64 prev = st ? (rec[st - 1] >> 17) : 0;
        --k;
        if (words && k < cap) {
            sr_conn_word w;
            w.slot = slot; w.cmd = slot / SR_FTR_PER_COMM; w.segment = 0; w.start = st; w.end = (u32)i + 1;
            w.dis = (u32)((r >> 17) - prev - pen);
            words[w0 + k] = w;
        }
        i = (int)st - 1;
    }
    n_words[s] = K;
    if (total) total[s] = last >> 17;
}

// ---- the grammar decoders' shared steps (K6g below, K13 further down) ------------------------------------------------
// Records are end keys D << kShift | copy << (kShift - 7) | ...: K6g's ekey (kShift = 17), K13's D << 7 | copy. They are
// read from L2 (ld.global.cg): other CTAs of the cluster wrote them, and this SM's L1 may hold a line of them from an
// earlier sequence.

// A sequence of no frames: no words, total 0 if state 0 is final, else ~0. The whole cluster leaves: no barrier, no
// remote store.
__device__ __forceinline__ void gram_empty(u32 rank, u32 s, u32 final_mask, u32 *n_words, u64 *total) {
    if (rank == 0 && threadIdx.x == 0) {
        if (n_words) n_words[s] = 0;
        if (total) total[s] = (final_mask & 1u) ? 0ull : ~0ull;
    }
}

// A sequence no path accepts: no words, total ~0.
__device__ __forceinline__ void gram_no_path(u32 s, u32 *n_words, u64 *total) {
    if (n_words) n_words[s] = 0;
    if (total) total[s] = ~0ull;
}

// Copy c's member from copy[c] = slot | state << 8 | src << 16: fills the state table cst of the ncand candidates, sets
// src and M (0: no copy or no member) and returns the template's slot.
__device__ __forceinline__ const unsigned char *copy_member(unsigned char *cst, const u32 *copy, u32 C, u32 ncand, u32 c,
                                                            const unsigned char *bank, u32 slot_stride, u32 &src, u32 &M) {
    for (u32 q = threadIdx.x; q < ncand; q += blockDim.x) cst[q] = q < C ? (unsigned char)((copy[q] >> 8) & 15u) : 0;
    const unsigned char *slot = bank;
    if (c < C) {
        const u32 cw = copy[c];
        src = cw >> 16;
        slot = bank + (size_t)(cw & 255u) * slot_stride;
        M = decode_frm(*reinterpret_cast<const u32 *>(slot), true);   // the host only makes copies of members
        if (M == kNoWalk) M = 0;
    }
    return slot;
}

// The entry term: the min over the candidates of the copies whose state is in src.
__device__ __forceinline__ u64 src_min(const u64 *buf, const unsigned char *cst, u32 ncand, u32 src, int lane) {
    u64 best = kEkeyNone;
    for (u32 q = lane; q < ncand; q += 32)
        if ((src >> cst[q]) & 1u) best = umin64(best, buf[q]);
    return warp_min(best);
}

// The per-state records: global warp gw reduces E_st over the candidates for the states st = gw (mod ncand), and its
// lane 0 hands each to store(st, E_st).
template <class Store>
__device__ __forceinline__ void state_records(const u64 *buf, const unsigned char *cst, u32 ncand, u32 S, u32 gw, int lane,
                                              Store store) {
    for (u32 st = gw; st < S; st += ncand) {
        u64 r = kEkeyNone;
        for (u32 q = lane; q < ncand; q += 32)
            if (cst[q] == st) r = umin64(r, buf[q]);
        r = warp_min(r);
        if (lane == 0) store(st, r);
    }
}

// argmin over the states of mask of E_s(f) (D only, ties to the lowest state); the records of frame f are at r
template <int kShift>
__device__ __forceinline__ u32 state_argmin(const u64 *r, u32 mask) {
    u32 best = 0;
    u64 bd = ~0ull;
    for (u32 s = 0; mask; ++s, mask >>= 1)
        if ((mask & 1u) && (__ldcg(r + s) >> kShift) < bd) { bd = __ldcg(r + s) >> kShift; best = s; }
    return best;
}

// The final state: the smallest E_s(N-1) over the final states, ties to the lowest state; S if none is reached. Its D
// goes to fd.
template <int kShift>
__device__ __forceinline__ u32 final_state(const u64 *R, u32 S, u32 N, u32 final_mask, u64 &fd) {
    u32 fs = S;
    u64 d = ~0ull;
    for (u32 st = 0; st < S; ++st) {
        const u64 r = __ldcg(R + (size_t)(N - 1) * S + st);
        if (((final_mask >> st) & 1u) && r != kEkeyNone && (r >> kShift) < d) { d = r >> kShift; fs = st; }
    }
    fd = d;
    return fs;
}

__global__ void __launch_bounds__(kConnWarps * 32, 2)
dtw_grammar_kernel(const s16 *__restrict__ feat, const u32 *__restrict__ frm_num,
                   const u32 *__restrict__ seq /* [.][3] first row, first record row, segment first frames (3 x 10 bits) */,
                   const unsigned char *__restrict__ bank, u32 slot_stride, const u32 *__restrict__ copy, u32 C, u32 S,
                   u32 final_mask, u32 penalty, u32 max_words, sr_conn_word *__restrict__ words /* or NULL */,
                   u32 *__restrict__ n_words /* or NULL */, u64 *__restrict__ total /* or NULL */, u64 *rec) {
    extern __shared__ __align__(128) unsigned char smem_raw[];
    cg::cluster_group cl = cg::this_cluster();
    const u32 nc = cl.num_blocks(), rank = cl.block_rank();
    const u32 s = blockIdx.x / nc;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    u64 *cand = reinterpret_cast<u64 *>(smem_raw + kSeqBytes + kConnWarps * kSlotBytes);   // [2][kConnCand]
    unsigned char *cst = reinterpret_cast<unsigned char *>(cand + 2 * kConnCand);          // [kConnCand] state of each copy
    const u32 N = frm_num[s];
    if (N == 0) return gram_empty(rank, s, final_mask, n_words, total);
    const u32 row0 = seq[3 * s], rec0 = seq[3 * s + 1], segs = seq[3 * s + 2];
    const u32 f0 = segs & 1023u, f1 = (segs >> 10) & 1023u, f2 = segs >> 20;
    const u32 ncand = nc * kConnWarps;
    const u32 c = rank * kConnWarps + warp;                // this warp's copy
    u32 src = 0;
    PRow b[4];
    u64 D[4];
    const u32 M = conn_prologue(cl, smem_raw, reinterpret_cast<const unsigned char *>(feat + (size_t)row0 * 12) - 4, N, b, D,
                                [&](u32 &M) { return copy_member(cst, copy, C, ncand, c, bank, slot_stride, src, M); });
    const u64 pen = penalty;
    u64 enter = (src & 1u) ? ((pen << 10) | 1023u) : kKeyInf;   // E_0(-1) + penalty: a word starting at frame 0 from state 0
    const u32 gw = rank * kConnWarps + warp;
    u64 *R = rec + (size_t)rec0 * S;
    for (u32 i = 0; i < N; ++i) {
        if (M && (i == f0 || i == f1 || i == f2)) {        // a segment's first frame: no word crosses the pause
#pragma unroll
            for (int k = 0; k < 4; ++k) D[k] = kKeyInf;
        }
        const u64 *buf = conn_frame(cl, nc, smem_raw, cand, i, M, enter, b, D, c);
        const u64 best = src_min(buf, cst, ncand, src, lane);
        enter = best == kEkeyNone ? kKeyInf : ((((best >> 17) + pen) << 10) | (u64)(1023u - (i + 1)));
        state_records(buf, cst, ncand, S, gw, lane, [&](u32 st, u64 r) { R[(size_t)i * S + st] = r; });
    }
    __threadfence();
    cl.sync();                                             // every CTA's records are written
    if (rank != 0 || threadIdx.x != 0) return;
    u64 fd;
    const u32 fs = final_state<17>(R, S, N, final_mask, fd);
    if (fs == S) return gram_no_path(s, n_words, total);
    // trace-back: the word ending at frame i in state st is [start, i + 1) of its copy, entered from the source state with
    // the smallest E(start - 1) (state 0 at start 0)
    u32 K = 0;
    for (int i = (int)N - 1, st = (int)fs; i >= 0;) {
        const u64 r = __ldcg(R + (size_t)i * S + st);
        const u32 b0 = (u32)(r & 1023u), cp = (u32)((r >> 10) & 127u);
        if (b0) st = (int)state_argmin<17>(R + (size_t)(b0 - 1) * S, copy[cp] >> 16);
        i = (int)b0 - 1;
        ++K;
    }
    u32 k = K;
    for (int i = (int)N - 1, st = (int)fs; i >= 0;) {
        const u64 r = __ldcg(R + (size_t)i * S + st);
        const u32 b0 = (u32)(r & 1023u), cp = (u32)((r >> 10) & 127u);
        u64 prev = 0;
        if (b0) {
            st = (int)state_argmin<17>(R + (size_t)(b0 - 1) * S, copy[cp] >> 16);
            prev = __ldcg(R + (size_t)(b0 - 1) * S + st) >> 17;
        }
        --k;
        if (words && k < max_words) {
            const u32 g = (f2 != kSegNone && b0 >= f2) ? 2u : (f1 != kSegNone && b0 >= f1) ? 1u : 0u;
            const u32 fb = g == 2 ? f2 : g == 1 ? f1 : f0;
            sr_conn_word w;
            w.slot = copy[cp] & 255u; w.cmd = w.slot / SR_FTR_PER_COMM; w.segment = g;
            w.start = b0 - fb; w.end = (u32)i + 1 - fb;
            w.dis = (u32)((r >> 17) - prev - pen);
            words[(size_t)s * max_words + k] = w;
        }
        i = (int)b0 - 1;
    }
    if (n_words) n_words[s] = K;
    if (total) total[s] = fd;
}

// rows [0, nf) of piece p's feature set -> long feature rows dst_row .. dst_row + nf - 1; pdst[p] = (dst_row, nf)
__global__ void __launch_bounds__(128)
conn_gather_kernel(const unsigned char *__restrict__ pf, const u32 *__restrict__ pdst, u32 P, s16 *__restrict__ feat) {
    for (u32 p = blockIdx.x; p < P; p += gridDim.x) {
        const u32 row = pdst[2 * p], nf = pdst[2 * p + 1];
        const u32 *src = reinterpret_cast<const u32 *>(pf + (size_t)p * kFtrBytes + 4);
        u32 *dst = reinterpret_cast<u32 *>(feat + (size_t)row * 12);
        for (u32 w = threadIdx.x; w < nf * 6; w += blockDim.x) dst[w] = src[w];
    }
}

// capture b's words: the decoded segments k = 0, 1, 2 (seq_of[b][k] = its sequence, 0xFFFFFFFF: none) in order, each
// word tagged with its segment; n_words = their sum, total = the saturating sum of the segments' totals
__global__ void __launch_bounds__(128)
conn_concat_kernel(const u32 *__restrict__ seq_of, const u32 *__restrict__ seq_off, const sr_conn_word *__restrict__ seq_words,
                   const u32 *__restrict__ seq_nw, const u64 *__restrict__ seq_total, u32 B, u32 max_words,
                   sr_conn_word *__restrict__ words, u32 *__restrict__ n_words, u64 *__restrict__ total) {
    const u32 b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= B) return;
    u32 cnt = 0;
    u64 tot = 0;
    for (int k = 0; k < 3; ++k) {
        const u32 sq = seq_of[3 * b + k];
        if (sq == 0xFFFFFFFFu) continue;
        const u32 nw = seq_nw[sq];
        const sr_conn_word *src = seq_words + seq_off[2 * sq + 1];
        for (u32 q = 0; q < nw && words; ++q) {
            if (cnt + q >= max_words) break;
            sr_conn_word w = src[q];
            w.segment = (u32)k;
            words[(size_t)b * max_words + cnt + q] = w;
        }
        cnt += nw;
        const u64 st = seq_total[sq];
        tot = (tot + st < tot) ? ~0ull : tot + st;
    }
    if (n_words) n_words[b] = cnt;
    if (total) total[b] = tot;
}

// C copies, 1 .. SR_GRAM_STATE_MAX states and nb sequences: what one grammar decoder launch takes
static bool gram_launch_ok(u32 C, u32 S, u32 nb) {
    return C <= SR_GRAM_COPY_MAX && S != 0 && S <= SR_GRAM_STATE_MAX && nb <= kSeqChunk;
}

// nb sequences, one cluster of ceil(n / kConnWarps) CTAs (one warp per slot or copy, at least one CTA) per sequence;
// clusters of more than 8 CTAs need the non-portable size
template <class... P, class... A>
static cudaError_t launch_clusters(void (*kernel)(P...), int smem, u32 nb, u32 n, cudaStream_t st, A &&...args) {
    const u32 nc = n ? (n + kConnWarps - 1) / kConnWarps : 1u;
    cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    if (e == cudaSuccess && nc > 8) e = cudaFuncSetAttribute(kernel, cudaFuncAttributeNonPortableClusterSizeAllowed, 1);
    if (e != cudaSuccess) return e;
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(nb * nc);
    cfg.blockDim = dim3(kConnWarps * 32);
    cfg.dynamicSmemBytes = smem;
    cfg.stream = st;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeClusterDimension;
    attr[0].val.clusterDim.x = nc;
    attr[0].val.clusterDim.y = 1;
    attr[0].val.clusterDim.z = 1;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    e = cudaLaunchKernelEx(&cfg, kernel, std::forward<A>(args)...);
    if (e != cudaSuccess) return e;
    return cudaGetLastError();
}

// sequences [b0, b0 + nb) against the bank's T <= SR_CONN_SLOT_MAX slots in one launch
cudaError_t launch_dtw_connected(const s16 *feat, u32 frm_stride, const u32 *frm_num, const u32 *seq_off, u32 b0, u32 nb,
                                 const void *bank, u32 T, u32 slot_stride, u32 penalty, u32 max_words, sr_conn_word *words,
                                 u32 *n_words, u64 *total, cudaStream_t st) {
    if (nb == 0) return cudaSuccess;
    if (T > SR_CONN_SLOT_MAX || nb > kSeqChunk) return cudaErrorInvalidValue;
    const s16 *f = seq_off ? feat : feat + (size_t)b0 * frm_stride * 12;
    return launch_clusters(dtw_connected_kernel, kConnSmem, nb, T, st, f, frm_stride, frm_num + b0,
                           seq_off ? seq_off + 2 * (size_t)b0 : nullptr, static_cast<const unsigned char *>(bank), T,
                           slot_stride, penalty, max_words, words && !seq_off ? words + (size_t)b0 * max_words : words,
                           n_words + b0, total ? total + b0 : nullptr);
}

// sequences [b0, b0 + nb) (the table seq gives each its first feature row, its first record row and its segments) against
// C <= SR_GRAM_COPY_MAX copies of the bank's slots in one launch. rec holds (last record row + 1) * S records; the caller
// chunks its sequences to bound it.
cudaError_t launch_dtw_grammar(const s16 *feat, const u32 *frm_num, const u32 *seq, u32 b0, u32 nb, const void *bank, u32 slot_stride,
                               const u32 *copy, u32 C, u32 S, u32 final_mask, u32 penalty, u32 max_words, sr_conn_word *words,
                               u32 *n_words, u64 *total, u64 *rec, cudaStream_t st) {
    if (nb == 0) return cudaSuccess;
    if (!gram_launch_ok(C, S, nb)) return cudaErrorInvalidValue;
    return launch_clusters(dtw_grammar_kernel, kGramSmem, nb, C, st, feat, frm_num + b0, seq + 3 * (size_t)b0,
                           static_cast<const unsigned char *>(bank), slot_stride, copy, C, S, final_mask, penalty, max_words,
                           words ? words + (size_t)b0 * max_words : nullptr, n_words ? n_words + b0 : nullptr,
                           total ? total + b0 : nullptr, rec);
}

// ---- K13: one grammar decode per long recording, across any number of segments (include/sr_long_grammar.h) -----------
// dtw_long_grammar_kernel is dtw_grammar_kernel's recurrence with three changes.
//  - Segments: the sequence owns segments k0 .. k0 + nk - 1 of a flat table (first feature row, frames <= 818; 0: nothing
//    to decode). Each segment with frames is staged in turn into the CTA's plane buffer, every within-word cell reset to
//    +inf, then decoded frame by frame; E, and with it the grammar state, carries across. A CTA restages its own buffer
//    only after the cluster barrier of the last frame of the segment before, which every warp passes after its last read
//    of that buffer; one CTA barrier then publishes the new planes.
//  - Keys, for D < 2^53 (headroom below): cells keep D << 10 | (1023 - start) with start the frame within the SEGMENT (a
//    word never crosses one, so the segment-relative order of starts is the sequence-relative one), +inf = 2^63. The end
//    cell is exchanged as D << 7 | copy (smallest D, ties to the lowest copy, as K6g's ekey orders them), and the start of
//    each copy's end cell, as a sequence-relative frame, goes to a second candidate array beside it.
//  - Records: per (frame, state) E_s(i) as D << 7 | copy (8 B) and its word's start frame (4 B), in two arrays.
// Headroom: a recording has at most F_max = (2^27 - 160) / 80 + 1 = 1 677 720 frames. A word of n frames has a path of at
// most n + 118 cells of get_dis <= 65 536, and there are at most F_max words, each adding the penalty (< 2^32):
// D < F_max * (119 * 65 536 + 2^32) < 2^52.7 < 2^53. So a cell key D << 10 stays below 2^63, and adding the row sums of one
// warp scan (< 128 * 2^26) to +inf = 2^63 stays below 2^64; the end key D << 7 | copy fits 60 bits.
constexpr int kLgSmem = kSeqBytes + kConnWarps * kSlotBytes + 2 * kConnCand * 8 + 2 * kConnCand * 4 + kConnCand;   // 52 792
constexpr u64 kLgInf = 1ull << 63;

// Frame li of segment-relative frames (its segment's first frame is sequence frame f0) of a warp whose copy's template has
// M frames: conn_column, then the end cell as D << 7 | idx to candidate idx, and its word's
// sequence-relative start to start candidate idx, of every CTA of the cluster; one cluster barrier.
__device__ __forceinline__ void lg_frame(cg::cluster_group &cl, u32 nc, const unsigned char *smem, u64 *cand, u32 *cstart,
                                         u32 li, u32 f0, u32 M, u64 enter, const PRow (&b)[4], u64 (&D)[4], u32 idx) {
    const int lane = threadIdx.x & 31;
    u64 mine = kEkeyNone;
    u32 mst = 0;
    if (M) {
        PRow a;
        load_row(a, smem, kSeqNrm, (int)li);               // broadcast read
        const u64 e = conn_column<kLgInf>(a, M, enter, b, D);
        if (e < kLgInf) {
            mine = ((e >> 10) << 7) | (u64)idx;
            mst = f0 + 1023u - (u32)(e & 1023u);
        }
    }
    if ((u32)lane < nc) {
        cl.map_shared_rank(cand, (unsigned)lane)[idx] = mine;
        cl.map_shared_rank(cstart, (unsigned)lane)[idx] = mst;
    }
    cl.sync();
}

__global__ void __launch_bounds__(kConnWarps * 32, 3)   // 80 registers: three CTAs per SM, as dtw_grammar_kernel
dtw_long_grammar_kernel(const s16 *__restrict__ feat, const u32 *__restrict__ seq /* [.][4] first segment, segments, frames, first record row */,
                        const u32 *__restrict__ seg_row, const u32 *__restrict__ seg_frm, const unsigned char *__restrict__ bank,
                        u32 slot_stride, const u32 *__restrict__ copy, u32 C, u32 S, u32 final_mask, u32 penalty, u32 max_words,
                        sr_conn_word *__restrict__ words /* or NULL */, u32 *__restrict__ n_words /* or NULL */,
                        u64 *__restrict__ total /* or NULL */, u64 *recD, u32 *recS) {
    extern __shared__ __align__(128) unsigned char smem_raw[];
    cg::cluster_group cl = cg::this_cluster();
    const u32 nc = cl.num_blocks(), rank = cl.block_rank();
    const u32 s = blockIdx.x / nc;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    u64 *cand = reinterpret_cast<u64 *>(smem_raw + kSeqBytes + kConnWarps * kSlotBytes);   // [2][kConnCand] end keys
    u32 *cstart = reinterpret_cast<u32 *>(cand + 2 * kConnCand);                            // [2][kConnCand] their starts
    unsigned char *cst = reinterpret_cast<unsigned char *>(cstart + 2 * kConnCand);         // [kConnCand] state of each copy
    const u32 k0 = seq[4 * s], nk = seq[4 * s + 1], N = seq[4 * s + 2], rec0 = seq[4 * s + 3];
    if (N == 0) return gram_empty(rank, s, final_mask, n_words, total);
    const u32 ncand = nc * kConnWarps;
    const u32 c = rank * kConnWarps + warp;                // this warp's copy
    u32 src = 0, M = 0;
    // copy_member's decode written out: through copy_member this kernel compiles to other SASS (77 registers), not timed
    const unsigned char *slot = bank;
    for (u32 q = threadIdx.x; q < ncand; q += blockDim.x) cst[q] = q < C ? (unsigned char)((copy[q] >> 8) & 15u) : 0;
    if (c < C) {
        const u32 cw = copy[c];
        src = cw >> 16;
        slot = bank + (size_t)(cw & 255u) * slot_stride;
        M = decode_frm(*reinterpret_cast<const u32 *>(slot), true);
        if (M == kNoWalk) M = 0;
    }
    unsigned char *tslot = smem_raw + kSeqBytes + warp * kSlotBytes;
    if (M) stage_planes(tslot, kNrm119, slot, (int)M, lane, 32);
    cl.sync();                                             // staging done, and every CTA of the cluster runs
    PRow b[4];
    u64 D[4];
#pragma unroll
    for (int k = 0; k < 4; ++k)
        if (M) load_row(b[k], tslot, kNrm119, lane * 4 + k < (int)M ? lane * 4 + k : 0);
    const u64 pen = penalty;
    u64 eb = (src & 1u) ? 0ull : ~0ull;                    // min over src of E_s(i - 1): E_0(-1) = 0
    const u32 gw = rank * kConnWarps + warp;
    u64 *R = recD + (size_t)rec0 * S;
    u32 *RS = recS + (size_t)rec0 * S;
    u32 gi = 0;                                            // sequence-relative frame
    for (u32 k = k0; k < k0 + nk; ++k) {
        const u32 F = seg_frm[k];
        if (F == 0) continue;
        stage_planes(smem_raw, kSeqNrm, reinterpret_cast<const unsigned char *>(feat + (size_t)seg_row[k] * 12) - 4, (int)F,
                     threadIdx.x, blockDim.x);
        __syncthreads();
#pragma unroll
        for (int q = 0; q < 4; ++q) D[q] = kLgInf;         // a segment's first frame: no word crosses the pause
        const u32 f0 = gi;
        for (u32 li = 0; li < F; ++li, ++gi) {
            const u64 enter = eb == ~0ull ? kLgInf : (((eb + pen) << 10) | (u64)(1023u - li));
            u64 *buf = cand + (gi & 1) * kConnCand;
            u32 *sb = cstart + (gi & 1) * kConnCand;
            lg_frame(cl, nc, smem_raw, buf, sb, li, f0, M, enter, b, D, c);
            const u64 best = src_min(buf, cst, ncand, src, lane);
            eb = best == kEkeyNone ? ~0ull : best >> 7;
            state_records(buf, cst, ncand, S, gw, lane, [&](u32 st, u64 r) {
                R[(size_t)gi * S + st] = r;
                RS[(size_t)gi * S + st] = r == kEkeyNone ? 0u : sb[r & 127u];   // and the start of its word
            });
        }
    }
    __threadfence();
    cl.sync();                                             // every CTA's records are written
    if (rank != 0 || threadIdx.x != 0) return;
    u64 fd;
    const u32 fs = final_state<7>(R, S, N, final_mask, fd);
    if (fs == S) return gram_no_path(s, n_words, total);
    // trace-back: the word ending at frame i in state st is [start, i + 1) of its copy, entered from the source state with
    // the smallest E(start - 1) (state 0 at start 0); frames map to (segment, frame within it) through the segment table
    u32 K = 0;
    for (long long i = (long long)N - 1, st = fs; i >= 0;) {
        const u64 r = __ldcg(R + (size_t)i * S + st);
        const u32 b0 = __ldcg(RS + (size_t)i * S + st);
        if (b0) st = state_argmin<7>(R + (size_t)(b0 - 1) * S, copy[r & 127u] >> 16);
        i = (long long)b0 - 1;
        ++K;
    }
    const u32 row0 = seg_row[k0];
    u32 kk = k0 + nk - 1, k = K;
    for (long long i = (long long)N - 1, st = fs; i >= 0;) {
        const u64 r = __ldcg(R + (size_t)i * S + st);
        const u32 b0 = __ldcg(RS + (size_t)i * S + st), cp = (u32)(r & 127u);
        u64 prev = 0;
        if (b0) {
            st = state_argmin<7>(R + (size_t)(b0 - 1) * S, copy[cp] >> 16);
            prev = __ldcg(R + (size_t)(b0 - 1) * S + st) >> 7;
        }
        --k;
        if (words && k < max_words) {
            while (seg_frm[kk] == 0 || seg_row[kk] - row0 > b0) --kk;
            const u32 fb = seg_row[kk] - row0;
            sr_conn_word w;
            w.slot = copy[cp] & 255u; w.cmd = w.slot / SR_FTR_PER_COMM; w.segment = kk - k0;
            w.start = b0 - fb; w.end = (u32)i + 1 - fb;
            w.dis = (u32)((r >> 7) - prev - pen);
            words[(size_t)s * max_words + k] = w;
        }
        i = (long long)b0 - 1;
    }
    if (n_words) n_words[s] = K;
    if (total) total[s] = fd;
}

// sequences [b0, b0 + nb) (seq: [.][4] first segment, segments, frames, first record row; seg_row / seg_frm: the flat
// segment table) against C <= SR_GRAM_COPY_MAX copies in one launch. recD / recS hold (last record row + 1) * S records;
// the caller cuts its sequences to bound them.
cudaError_t launch_dtw_long_grammar(const s16 *feat, const u32 *seq, u32 b0, u32 nb, const u32 *seg_row, const u32 *seg_frm,
                                    const void *bank, u32 slot_stride, const u32 *copy, u32 C, u32 S, u32 final_mask, u32 penalty,
                                    u32 max_words, sr_conn_word *words, u32 *n_words, u64 *total, u64 *recD, u32 *recS,
                                    cudaStream_t st) {
    if (nb == 0) return cudaSuccess;
    if (!gram_launch_ok(C, S, nb)) return cudaErrorInvalidValue;
    return launch_clusters(dtw_long_grammar_kernel, kLgSmem, nb, C, st, feat, seq + 4 * (size_t)b0, seg_row, seg_frm,
                           static_cast<const unsigned char *>(bank), slot_stride, copy, C, S, final_mask, penalty, max_words,
                           words ? words + (size_t)b0 * max_words : nullptr, n_words ? n_words + b0 : nullptr,
                           total ? total + b0 : nullptr, recD, recS);
}

cudaError_t launch_conn_gather(const void *pf, const u32 *pdst, u32 P, s16 *feat, int num_sms, cudaStream_t st) {
    if (P == 0) return cudaSuccess;
    const u32 grid = P < (u32)num_sms * 16u ? P : (u32)num_sms * 16u;
    conn_gather_kernel<<<grid, 128, 0, st>>>(static_cast<const unsigned char *>(pf), pdst, P, feat);
    return cudaGetLastError();
}

cudaError_t launch_conn_concat(const u32 *seq_of, const u32 *seq_off, const sr_conn_word *seq_words, const u32 *seq_nw,
                               const u64 *seq_total, u32 B, u32 max_words, sr_conn_word *words, u32 *n_words, u64 *total,
                               cudaStream_t st) {
    if (B == 0) return cudaSuccess;
    conn_concat_kernel<<<(B + 127) / 128, 128, 0, st>>>(seq_of, seq_off, seq_words, seq_nw, seq_total, B, max_words, words,
                                                       n_words, total);
    return cudaGetLastError();
}

}  // namespace srk
