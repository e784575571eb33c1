// sr_dtw_grammar.cu -- K6g: connected words under a finite-state grammar, one-pass DP over a network of template copies
// (Ney 1984; EXTENSION, checked against this project's own CPU restatement and plain Python references, parity unpinned).
//
// dtw_grammar_kernel is dtw_connected_kernel (sr_dtw_connected.cu) with the bank replaced by the grammar's COPIES: a copy
// c = (state s', member slot t) exists when some arc into s' carries cmd(t), and enters from src(c), the states with such an
// arc. The host numbers the copies state-major, then by slot, and hands the kernel one word per copy,
//   copy[c] = slot | state << 8 | src << 16.
// One thread-block CLUSTER per sequence, one WARP per copy (kGramWarps per CTA, ceil(C / kGramWarps) <= 16 CTAs). A warp
// holds its template's rows in registers and advances one input frame per step exactly as the K6 warp does: one warp scan
// of the lanes' (min,+) maps and a serial fix-up pass over the 64-bit cell keys D << 10 | (1023 - start). After each
// frame every warp sends its end cell as ekey = D << 17 | copy << 10 | start to every CTA of the cluster over DSMEM, one
// cluster barrier follows (candidates double-buffered by frame parity, as in K6), and then
//   - each warp reduces only the candidates whose copy's state is in its own src mask: min_{s in src} E_s(i) + P is the
//     coupling term of its cell j = 0 at frame i + 1 (the state of every copy is kept in a shared byte table);
//   - global warp g reduces E_s(i) for the states s = g (mod warps in the cluster) and stores it, as an ekey, to the
//     sequence's record rows in global memory: rec[(rec0 + i) * S + s].
// At the first frame of a later segment every within-word cell is reset to +inf, so no word crosses the pause, while E and
// with it the grammar state carry over. After the last frame one lane of rank 0 picks the final state and traces back
// through the records, writing each word with its segment and segment-relative frames.
//
// Headroom is K6's: D < 2^42 (at most 818 frames in one sequence, every word adds the penalty < 2^32), the copy index
// takes K6's 7-bit slot field.
#include <cooperative_groups.h>
#include "sr_dtw_core.cuh"

namespace cg = cooperative_groups;

namespace srk {

constexpr int kGramWarps = 8;                              // copies per CTA
constexpr int kGramCluster = 16;                           // CTAs per cluster at most: SR_GRAM_COPY_MAX = 128 copies
constexpr int kGramCand = kGramWarps * kGramCluster;       // candidates per frame buffer
constexpr u32 kGramFrm = SR_CONN_FRM_MAX;                  // 818
constexpr u32 kGSeqNrm = kGramFrm * 24;                    // norm offset of the sequence's byte-plane slot
constexpr int kGSeqBytes = kGramFrm * 28;                  // 22 904
constexpr int kGramSmem = kGSeqBytes + kGramWarps * kSlotBytes + 2 * kGramCand * 8 + kGramCand;   // 51 768
constexpr u64 kGKeyInf = 1ull << 62;
constexpr u64 kGEkeyNone = ~0ull;
constexpr u32 kSegNone = 1023u;                            // segment field of a segment without frames
static_assert(kGramWarps * kGramCluster == SR_GRAM_COPY_MAX, "one warp per copy");
static_assert(kGramFrm < kSegNone, "start frames and segment first frames are 10-bit fields");

__device__ __forceinline__ u64 gmin64(u64 a, u64 b) { return a < b ? a : b; }

// argmin over the states of mask of E_s(f) (D only, ties to the lowest state); the records of frame f are at r
__device__ __forceinline__ u32 gram_src(const u64 *r, u32 mask) {
    u32 best = 0;
    u64 bd = ~0ull;
    for (u32 s = 0; mask; ++s, mask >>= 1)
        if ((mask & 1u) && (__ldcg(r + s) >> 17) < bd) { bd = __ldcg(r + s) >> 17; best = s; }
    return best;
}

__global__ void __launch_bounds__(kGramWarps * 32, 2)
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
    unsigned char *sq = smem_raw;
    unsigned char *tslot = sq + kGSeqBytes + warp * kSlotBytes;
    u64 *cand = reinterpret_cast<u64 *>(sq + kGSeqBytes + kGramWarps * kSlotBytes);   // [2][kGramCand]
    unsigned char *cst = reinterpret_cast<unsigned char *>(cand + 2 * kGramCand);    // [kGramCand] state of each copy
    const u32 N = frm_num[s];
    if (N == 0) {                                          // the whole cluster leaves: no barrier, no remote store
        if (rank == 0 && threadIdx.x == 0) {
            if (n_words) n_words[s] = 0;
            if (total) total[s] = (final_mask & 1u) ? 0ull : ~0ull;
        }
        return;
    }
    const u32 row0 = seq[3 * s], rec0 = seq[3 * s + 1], segs = seq[3 * s + 2];
    const u32 f0 = segs & 1023u, f1 = (segs >> 10) & 1023u, f2 = segs >> 20;
    stage_planes(sq, kGSeqNrm, reinterpret_cast<const unsigned char *>(feat + (size_t)row0 * 12) - 4, (int)N, threadIdx.x,
                 blockDim.x);
    const u32 ncand = nc * kGramWarps;
    for (u32 q = threadIdx.x; q < ncand; q += blockDim.x) cst[q] = q < C ? (unsigned char)((copy[q] >> 8) & 15u) : 0;
    const u32 c = rank * kGramWarps + warp;                // this warp's copy
    u32 M = 0, src = 0;                                    // M = 0: no copy, never walked
    if (c < C) {
        const u32 cw = copy[c];
        src = cw >> 16;
        const unsigned char *slot = bank + (size_t)(cw & 255u) * slot_stride;
        M = decode_frm(*reinterpret_cast<const u32 *>(slot), SR_DTW_CHECK_SIGN);   // the host only makes copies of members
        if (M == kNoWalk) M = 0;
        if (M) stage_planes(tslot, kNrm119, slot, (int)M, lane, 32);
    }
    cl.sync();                                             // staging done, and every CTA of the cluster runs
    const int j0 = lane * 4;
    PRow b[4];
    u64 D[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        if (M) load_row(b[k], tslot, kNrm119, j0 + k < (int)M ? j0 + k : 0);
        D[k] = kGKeyInf;
    }
    const u64 pen = penalty;
    u64 enter = (src & 1u) ? ((pen << 10) | 1023u) : kGKeyInf;   // E_0(-1) + penalty: a word starting at frame 0 from state 0
    const u32 gw = rank * kGramWarps + warp;
    u64 *R = rec + (size_t)rec0 * S;
    const int lend = ((int)M - 1) >> 2, kend = ((int)M - 1) & 3;
    for (u32 i = 0; i < N; ++i) {
        u64 mine = kGEkeyNone;
        if (M) {
            if (i == f0 || i == f1 || i == f2) {            // a segment's first frame: no word crosses the pause
#pragma unroll
                for (int k = 0; k < 4; ++k) D[k] = kGKeyInf;
            }
            PRow a;
            load_row(a, sq, kGSeqNrm, (int)i);             // broadcast read
            u64 dg = __shfl_up_sync(0xFFFFFFFFu, D[3], 1); // D(i-1, j0-1)
            if (lane == 0) dg = kGKeyInf;
            u64 dk[4], A[4];
            bool valid[4];
            u64 x = kGKeyInf, sum = 0;                     // serial pass for an incoming +inf
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                const int j = j0 + k;
                valid[k] = j < (int)M;
                dk[k] = (u64)pdist(a, b[k]) << 10;
                A[k] = gmin64(D[k], j == 0 ? enter : dg);
                dg = D[k];
                x = valid[k] ? gmin64(dk[k] + gmin64(A[k], x), kGKeyInf) : kGKeyInf;
                sum += dk[k];
            }
            u64 fa = sum, fb = x;                          // inclusive composition of the lanes' maps min(x + fa, fb)
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const u64 pa = __shfl_up_sync(0xFFFFFFFFu, fa, o), pb = __shfl_up_sync(0xFFFFFFFFu, fb, o);
                if (lane >= o) { fb = gmin64(gmin64(pb + fa, fb), kGKeyInf); fa += pa; }
            }
            x = __shfl_up_sync(0xFFFFFFFFu, gmin64(kGKeyInf + fa, fb), 1);
            if (lane == 0) x = kGKeyInf;
            x = gmin64(x, kGKeyInf);
#pragma unroll
            for (int k = 0; k < 4; ++k) {                  // serial fix-up with the true incoming x = D(i, j-1)
                x = valid[k] ? gmin64(dk[k] + gmin64(A[k], x), kGKeyInf) : kGKeyInf;
                D[k] = x;
            }
            u64 e = D[0];
#pragma unroll
            for (int k = 1; k < 4; ++k) if (k == kend) e = D[k];
            e = __shfl_sync(0xFFFFFFFFu, e, lend);
            if (e < kGKeyInf) mine = ((e >> 10) << 17) | ((u64)c << 10) | (u64)(1023u - (u32)(e & 1023u));
        }
        u64 *buf = cand + (i & 1) * kGramCand;
        if ((u32)lane < nc) cl.map_shared_rank(buf, (unsigned)lane)[c] = mine;
        cl.sync();
        u64 best = kGEkeyNone;                             // min over the copies of the states in src: the entry term
        for (u32 q = lane; q < ncand; q += 32)
            if ((src >> cst[q]) & 1u) best = gmin64(best, buf[q]);
#pragma unroll
        for (int o = 16; o; o >>= 1) best = gmin64(best, __shfl_xor_sync(0xFFFFFFFFu, best, o));
        enter = best == kGEkeyNone ? kGKeyInf : ((((best >> 17) + pen) << 10) | (u64)(1023u - (i + 1)));
        for (u32 st = gw; st < S; st += ncand) {           // the records E_st(i) this warp owns
            u64 r = kGEkeyNone;
            for (u32 q = lane; q < ncand; q += 32)
                if (cst[q] == st) r = gmin64(r, buf[q]);
#pragma unroll
            for (int o = 16; o; o >>= 1) r = gmin64(r, __shfl_xor_sync(0xFFFFFFFFu, r, o));
            if (lane == 0) R[(size_t)i * S + st] = r;
        }
    }
    __threadfence();
    cl.sync();                                             // every CTA's records are written
    if (rank != 0 || threadIdx.x != 0) return;
    // records are read from L2 (ld.global.cg): other CTAs of the cluster wrote them, and this SM's L1 may hold a line of
    // them from an earlier sequence. The final state: the smallest E_s(N-1) over final states, ties to the lowest state
    u32 fs = S;
    u64 fd = ~0ull;
    for (u32 st = 0; st < S; ++st) {
        const u64 r = __ldcg(R + (size_t)(N - 1) * S + st);
        if (((final_mask >> st) & 1u) && r != kGEkeyNone && (r >> 17) < fd) { fd = r >> 17; fs = st; }
    }
    if (fs == S) {                                         // no accepting path
        if (n_words) n_words[s] = 0;
        if (total) total[s] = ~0ull;
        return;
    }
    // trace-back: the word ending at frame i in state st is [start, i + 1) of its copy, entered from the source state with
    // the smallest E(start - 1) (state 0 at start 0)
    u32 K = 0;
    for (int i = (int)N - 1, st = (int)fs; i >= 0;) {
        const u64 r = __ldcg(R + (size_t)i * S + st);
        const u32 b0 = (u32)(r & 1023u), cp = (u32)((r >> 10) & 127u);
        if (b0) st = (int)gram_src(R + (size_t)(b0 - 1) * S, copy[cp] >> 16);
        i = (int)b0 - 1;
        ++K;
    }
    u32 k = K;
    for (int i = (int)N - 1, st = (int)fs; i >= 0;) {
        const u64 r = __ldcg(R + (size_t)i * S + st);
        const u32 b0 = (u32)(r & 1023u), cp = (u32)((r >> 10) & 127u);
        u64 prev = 0;
        if (b0) {
            st = (int)gram_src(R + (size_t)(b0 - 1) * S, copy[cp] >> 16);
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

// sequences [b0, b0 + nb) (the table seq gives each its first feature row, its first record row and its segments) against
// C <= SR_GRAM_COPY_MAX copies of the bank's slots in one launch: one cluster of ceil(C / kGramWarps) CTAs per sequence.
// rec holds (last record row + 1) * S records; the caller chunks its sequences to bound it.
cudaError_t launch_dtw_grammar(const s16 *feat, const u32 *frm_num, const u32 *seq, u32 b0, u32 nb, const void *bank, u32 slot_stride,
                               const u32 *copy, u32 C, u32 S, u32 final_mask, u32 penalty, u32 max_words, sr_conn_word *words,
                               u32 *n_words, u64 *total, u64 *rec, cudaStream_t st) {
    if (nb == 0) return cudaSuccess;
    if (C > SR_GRAM_COPY_MAX || S == 0 || S > SR_GRAM_STATE_MAX || nb > kSeqChunk) return cudaErrorInvalidValue;
    const u32 nc = C ? (C + kGramWarps - 1) / kGramWarps : 1u;
    cudaError_t e = cudaFuncSetAttribute(dtw_grammar_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kGramSmem);
    if (e == cudaSuccess && nc > 8) e = cudaFuncSetAttribute(dtw_grammar_kernel, cudaFuncAttributeNonPortableClusterSizeAllowed, 1);
    if (e != cudaSuccess) return e;
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(nb * nc);
    cfg.blockDim = dim3(kGramWarps * 32);
    cfg.dynamicSmemBytes = kGramSmem;
    cfg.stream = st;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeClusterDimension;
    attr[0].val.clusterDim.x = nc;
    attr[0].val.clusterDim.y = 1;
    attr[0].val.clusterDim.z = 1;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    e = cudaLaunchKernelEx(&cfg, dtw_grammar_kernel, feat, frm_num + b0, seq + 3 * (size_t)b0,
                           static_cast<const unsigned char *>(bank), slot_stride, copy, C, S, final_mask, penalty, max_words,
                           words ? words + (size_t)b0 * max_words : nullptr, n_words ? n_words + b0 : nullptr,
                           total ? total + b0 : nullptr, rec);
    if (e != cudaSuccess) return e;
    return cudaGetLastError();
}

}  // namespace srk
