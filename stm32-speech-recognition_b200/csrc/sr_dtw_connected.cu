// sr_dtw_connected.cu -- K6: connected words by one-pass DP over the template bank (one-stage DTW, Ney 1984)
// (EXTENSION: the reference decodes one word per VAD segment; checked against this project's own CPU restatement and
// plain Python references, parity unpinned).
//
// dtw_connected_kernel: one thread-block CLUSTER per feature sequence, one WARP per bank slot (kConnWarps slots per CTA,
// up to kConnCluster CTAs per cluster). A warp holds its template's rows in registers, lane l owning columns 4l .. 4l+3
// as in dtw_wide_kernel / dtw_align_kernel, and advances one input frame per step: one warp scan of the lanes' (min,+)
// maps and a serial fix-up pass write the template's column of D for that frame. Cells are 64-bit keys
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
// Headroom: a word's path has at most len + M - 1 <= 818 + 118 cells of get_dis <= 65 535, and at most 818 words each add
// the penalty (< 2^32): D < 119 * 818 * 65 536 + 818 * 2^32 < 2^42, so D << 17 | slot << 10 | start fits 59 bits and
// D << 10 plus the row sums of one warp scan (< 128 * 2^26) stays below the infinity 2^62.
//
// conn_gather_kernel copies the rows of get_mfcc pieces into their long feature rows; conn_concat_kernel joins the words
// of the segments of one capture (sr_recognise_connected_batch).
#include <cooperative_groups.h>
#include "sr_dtw_core.cuh"

namespace cg = cooperative_groups;

namespace srk {

constexpr int kConnWarps = 8;                              // bank slots per CTA
constexpr int kConnCluster = 16;                           // CTAs per cluster at most: SR_CONN_SLOT_MAX = 128 slots
constexpr int kConnCand = kConnWarps * kConnCluster;       // candidates per frame buffer
constexpr u32 kConnFrm = SR_CONN_FRM_MAX;                  // 818
constexpr u32 kSeqNrm = kConnFrm * 24;                     // norm offset of the sequence's byte-plane slot
constexpr int kSeqBytes = kConnFrm * 28;                   // 22 904
constexpr int kConnSmem = kSeqBytes + kConnWarps * kSlotBytes + 2 * kConnCand * 8 + kConnFrm * 8;   // 58 184
constexpr u64 kKeyInf = 1ull << 62;
constexpr u64 kEkeyNone = ~0ull;
static_assert(kConnWarps * kConnCluster == SR_CONN_SLOT_MAX, "one warp per slot");
static_assert(kConnFrm < 1024, "start frames are 10-bit fields of the keys");

__device__ __forceinline__ u64 umin64(u64 a, u64 b) { return a < b ? a : b; }

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
    unsigned char *seq = smem_raw;
    unsigned char *tslot = seq + kSeqBytes + warp * kSlotBytes;
    u64 *cand = reinterpret_cast<u64 *>(seq + kSeqBytes + kConnWarps * kSlotBytes);   // [2][kConnCand]
    u64 *rec = cand + 2 * kConnCand;                                                   // [kConnFrm] E(i) as ekey
    const u32 N = frm_num[s];
    if (N == 0) {                                          // the whole cluster leaves: no barrier, no remote store
        if (rank == 0 && threadIdx.x == 0) {
            n_words[s] = 0;
            if (total) total[s] = 0;
        }
        return;
    }
    const size_t row0 = seq_off ? seq_off[2 * s] : (size_t)s * frm_stride;
    // the sequence's rows as byte planes (stage_planes reads row r at src + 4 + 24 r: a header-less row array shifted by 4)
    stage_planes(seq, kSeqNrm, reinterpret_cast<const unsigned char *>(feat + row0 * 12) - 4, (int)N, threadIdx.x, blockDim.x);
    const u32 t = rank * kConnWarps + warp;                // this warp's bank slot
    u32 M = 0;                                             // 0: not a member, never walked
    if (t < T) {
        const unsigned char *slot = bank + (size_t)t * slot_stride;
        const u32 frm = decode_frm(*reinterpret_cast<const u32 *>(slot), SR_DTW_CHECK_SIGN);
        if (frm != kNoWalk) M = frm;
        if (M) stage_planes(tslot, kNrm119, slot, (int)M, lane, 32);
    }
    cl.sync();                                             // staging done, and every CTA of the cluster runs
    const int j0 = lane * 4;
    PRow b[4];
    u64 D[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        if (M) load_row(b[k], tslot, kNrm119, j0 + k < (int)M ? j0 + k : 0);
        D[k] = kKeyInf;
    }
    const u64 pen = penalty;
    u64 enter = (pen << 10) | 1023u;                       // E(-1) + penalty, a word starting at frame 0
    const u32 ncand = nc * kConnWarps;
    const int lend = ((int)M - 1) >> 2, kend = ((int)M - 1) & 3;
    for (u32 i = 0; i < N; ++i) {
        u64 mine = kEkeyNone;
        if (M) {
            PRow a;
            load_row(a, seq, kSeqNrm, (int)i);             // broadcast read
            u64 dg = __shfl_up_sync(0xFFFFFFFFu, D[3], 1); // D(i-1, j0-1)
            if (lane == 0) dg = kKeyInf;
            u64 dk[4], A[4];
            bool valid[4];
            u64 x = kKeyInf, sum = 0;                      // serial pass for an incoming +inf
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                const int j = j0 + k;
                valid[k] = j < (int)M;
                dk[k] = (u64)pdist(a, b[k]) << 10;
                A[k] = umin64(D[k], j == 0 ? enter : dg);
                dg = D[k];
                x = valid[k] ? umin64(dk[k] + umin64(A[k], x), kKeyInf) : kKeyInf;
                sum += dk[k];
            }
            u64 fa = sum, fb = x;                          // inclusive composition of the lanes' maps min(x + fa, fb)
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const u64 pa = __shfl_up_sync(0xFFFFFFFFu, fa, o), pb = __shfl_up_sync(0xFFFFFFFFu, fb, o);
                if (lane >= o) { fb = umin64(umin64(pb + fa, fb), kKeyInf); fa += pa; }
            }
            x = __shfl_up_sync(0xFFFFFFFFu, umin64(kKeyInf + fa, fb), 1);
            if (lane == 0) x = kKeyInf;
            x = umin64(x, kKeyInf);
#pragma unroll
            for (int k = 0; k < 4; ++k) {                  // serial fix-up with the true incoming x = D(i, j-1)
                x = valid[k] ? umin64(dk[k] + umin64(A[k], x), kKeyInf) : kKeyInf;
                D[k] = x;
            }
            u64 e = D[0];
#pragma unroll
            for (int k = 1; k < 4; ++k) if (k == kend) e = D[k];
            e = __shfl_sync(0xFFFFFFFFu, e, lend);
            if (e < kKeyInf) mine = ((e >> 10) << 17) | ((u64)t << 10) | (u64)(1023u - (u32)(e & 1023u));
        }
        u64 *buf = cand + (i & 1) * kConnCand;
        if ((u32)lane < nc) cl.map_shared_rank(buf, (unsigned)lane)[t] = mine;
        cl.sync();
        u64 best = kEkeyNone;
        for (u32 q = lane; q < ncand; q += 32) best = umin64(best, buf[q]);
#pragma unroll
        for (int o = 16; o; o >>= 1) best = umin64(best, __shfl_xor_sync(0xFFFFFFFFu, best, o));
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

// sequences [b0, b0 + nb) against the bank's T <= SR_CONN_SLOT_MAX slots in one launch: one cluster of
// ceil(T / kConnWarps) CTAs per sequence
cudaError_t launch_dtw_connected(const s16 *feat, u32 frm_stride, const u32 *frm_num, const u32 *seq_off, u32 b0, u32 nb,
                                 const void *bank, u32 T, u32 slot_stride, u32 penalty, u32 max_words, sr_conn_word *words,
                                 u32 *n_words, u64 *total, cudaStream_t st) {
    if (nb == 0) return cudaSuccess;
    if (T > SR_CONN_SLOT_MAX || nb > kSeqChunk) return cudaErrorInvalidValue;
    const u32 nc = T ? (T + kConnWarps - 1) / kConnWarps : 1u;
    cudaError_t e = cudaFuncSetAttribute(dtw_connected_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kConnSmem);
    if (e == cudaSuccess && nc > 8) e = cudaFuncSetAttribute(dtw_connected_kernel, cudaFuncAttributeNonPortableClusterSizeAllowed, 1);
    if (e != cudaSuccess) return e;
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(nb * nc);
    cfg.blockDim = dim3(kConnWarps * 32);
    cfg.dynamicSmemBytes = kConnSmem;
    cfg.stream = st;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeClusterDimension;
    attr[0].val.clusterDim.x = nc;
    attr[0].val.clusterDim.y = 1;
    attr[0].val.clusterDim.z = 1;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    const s16 *f = seq_off ? feat : feat + (size_t)b0 * frm_stride * 12;
    e = cudaLaunchKernelEx(&cfg, dtw_connected_kernel, f, frm_stride, frm_num + b0, seq_off ? seq_off + 2 * (size_t)b0 : nullptr,
                           static_cast<const unsigned char *>(bank), T, slot_stride, penalty, max_words,
                           words && !seq_off ? words + (size_t)b0 * max_words : words, n_words + b0,
                           total ? total + b0 : nullptr);
    if (e != cudaSuccess) return e;
    return cudaGetLastError();
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
