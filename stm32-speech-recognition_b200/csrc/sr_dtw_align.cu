// sr_dtw_align.cu -- K3p: the banded DP of K3 with its optimal warping path, and DTW barycentre averaging of bank groups
// (EXTENSION: the reference has no DP; checked against this project's own CPU restatement and plain numpy references,
// parity unpinned).
//
// dtw_align_kernel: one WARP per (input, template) pair, in the whole-row form of dtw_wide_kernel for EVERY r (the cost
// does not depend on r, the band only masks cells): lane l owns columns 4l .. 4l+3, the template's four rows stay in
// registers, and each row is one dp_column step (sr_dtw_core.cuh): a warp scan of the lanes' (min,+) maps and a serial
// fix-up pass. During the fix-up pass each cell records which neighbour its minimum came from, 2 bits (0 diagonal,
// 1 (i, j-1), 2 (i-1, j)), ties in that order: one byte per lane per row, 119 x 32 B per warp in shared memory. After
// the last row lane 0 traces back from
// (I-1, M-1) to (0, 0) (at most I + M - 1 <= 237 steps) and the warp writes the path forward, (i, j) byte pairs, padded
// with 0xFF. Pairs come as a list over two base pointers with their own strides (bank slots, v_ftr_tag rows), so the one
// kernel serves sr_dtw_path_batch and every pass of sr_average_bank; in "pick" mode the template of a pair is the
// anchor of its group, chosen in the kernel from the group's K x K anchor scores.
//
// average_update_kernel: one CTA per group; sums every aligned member's frames into the template columns their paths
// visit (shared-memory integer atomics: the sums do not depend on order), then C[j] = sum[j] / cnt[j] truncated.
#include "sr_dtw_core.cuh"

namespace srk {

constexpr int kAlignWarps = 8;                            // 8 x 10 960 B of shared memory: two CTAs per SM
constexpr int kAlignCells = 4;                            // columns per lane: 32 x 4 = 128 >= 119
constexpr int kPathMax = 2 * kMaxFrm - 1;                 // 237 = I + M - 1 at most
constexpr int kChoiceBytes = kMaxFrm * 32;                // one byte per lane per row
constexpr int kPathBuf = 480;                             // 237 u16 points, rounded up
constexpr int kAlignWarpBytes = 2 * kSlotBytes + kChoiceBytes + kPathBuf;
constexpr s32 kAlignInf = 0x3FFFFFFF;                     // the s32 headroom of dp_column (sr_dtw_core.cuh)

struct AlignPair { u32 in, tpl, out; };

// the anchor of a group: the member k with the smallest sum over the other members l of S(l -> k), the u64 sum counting
// SR_DIS_ERR as 0xFFFFFFFF, ties to the lowest k. S is the group's K x K block (S[l * K + k]), mask its members. Lane k
// scores candidate k; every lane returns the winner.
__device__ __forceinline__ u32 pick_anchor(const u32 *S, u32 K, u32 mask, int lane) {
    u64 key = ~0ull;
    if ((u32)lane < K && ((mask >> lane) & 1u)) {
        u64 s = 0;
        for (u32 l = 0; l < K; ++l)
            if (l != (u32)lane && ((mask >> l) & 1u)) s += S[l * K + lane];
        key = (s << 5) | (u64)lane;                       // s < 32 * 2^32: fits above the 5 index bits
    }
#pragma unroll
    for (int o = 16; o; o >>= 1) { const u64 other = __shfl_xor_sync(0xFFFFFFFFu, key, o); key = other < key ? other : key; }
    return (u32)(key & 31u);
}

// The DP of one staged pair (I, M >= 1, within the 2:1 guard) at radius r <= 118; returns D(I-1, M-1) or kAlignInf when
// the end cell is unreachable. With choice != NULL every row's predecessor choices are written there.
__device__ __forceinline__ s32 align_dp(int I, int M, int r, const unsigned char *uslot, const unsigned char *tslot,
                                        u8 *choice, int lane) {
    const int j0 = lane * kAlignCells;
    PRow b[kAlignCells];
    s32 D[kAlignCells];
#pragma unroll
    for (int k = 0; k < kAlignCells; ++k) {
        load_row(b[k], tslot, kNrm119, j0 + k < M ? j0 + k : 0);
        D[k] = kAlignInf;
    }
    for (int i = 0; i < I; ++i) {
        const int c = (i * M) / I, lo = max(c - r, 0), hi = min(c + r, M - 1);
        PRow a;
        load_row(a, uslot, kNrm119, i);                              // broadcast read
        bool dfirst[kAlignCells];
        u32 byte = 0;
        dp_column<s32, kAlignInf>(D, lane, [&](int k, s32 up, s32 dg, s32 &d, s32 &A, bool &valid) {
            const int j = j0 + k;
            valid = j >= lo && j <= hi;
            d = valid ? (s32)pdist(a, b[k]) : 0;
            dfirst[k] = dg <= up;                                    // the diagonal is at least as good as (i-1, j)
            A = i == 0 ? (j == 0 ? 0 : kAlignInf) : min(up, dg);
        }, [&](int k, s32 A, s32 x) {
            // minimum of diagonal, (i, j-1), (i-1, j), ties in that order
            const u32 ch = dfirst[k] ? (A <= x ? 0u : 1u) : (x <= A ? 1u : 2u);
            byte |= ch << (2 * k);
        });
        if (choice) choice[i * 32 + lane] = (u8)byte;
    }
    const s32 fin = dp_end(D, (M - 1) & (kAlignCells - 1), (M - 1) / kAlignCells);
    return fin < kAlignInf / 2 ? fin : kAlignInf;
}

__global__ void __launch_bounds__(kAlignWarps * 32, 2)
dtw_align_kernel(const unsigned char *__restrict__ in_base, u32 in_stride, const unsigned char *__restrict__ tpl_base,
                 u32 tpl_stride, const AlignPair *__restrict__ pairs /* NULL: pair p = (p, p, p) */, u32 n, int r,
                 u8 *__restrict__ path /* [.][kPathMax][2] or NULL */, u32 *__restrict__ path_len /* or NULL */,
                 u32 *__restrict__ dis /* or NULL */,
                 // pick mode (pick_S != NULL): pair.tpl is a group g, the template its anchor: slot g*K + anchor of the
                 // input bank; the warp aligning the anchor itself copies it to tpl_out[g] and writes anchor_out[g]
                 const u32 *__restrict__ pick_S, const u32 *__restrict__ mask, u32 K, unsigned char *__restrict__ tpl_out,
                 u32 *__restrict__ anchor_out) {
    extern __shared__ __align__(128) unsigned char smem_raw[];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    unsigned char *uslot = smem_raw + (size_t)warp * kAlignWarpBytes;
    unsigned char *tslot = uslot + kSlotBytes;
    u8 *choice = tslot + kSlotBytes;
    u16 *pbuf = reinterpret_cast<u16 *>(choice + kChoiceBytes);
    const bool want_path = path || path_len;
    for (u32 p = blockIdx.x * kAlignWarps + warp; p < n; p += gridDim.x * kAlignWarps) {
        const AlignPair pr = pairs ? pairs[p] : AlignPair{p, p, p};
        const unsigned char *uf = in_base + (size_t)pr.in * in_stride;
        u32 anchor = 0;
        const unsigned char *tf;
        if (pick_S) {
            anchor = pick_anchor(pick_S + (size_t)pr.tpl * K * K, K, mask[pr.tpl], lane);
            tf = in_base + ((size_t)pr.tpl * K + anchor) * in_stride;
        } else {
            tf = tpl_base + (size_t)pr.tpl * tpl_stride;
        }
        const u32 Iraw = decode_frm(*reinterpret_cast<const u32 *>(uf), false), Mraw = decode_frm(*reinterpret_cast<const u32 *>(tf), false);
        const bool walks = Iraw >= 1 && pair_walks(Iraw, Mraw, true);
        const int I = (int)Iraw, M = (int)Mraw;
        __syncwarp();                                                // the previous pair's readers are done
        if (walks) {
            stage_planes(uslot, kNrm119, uf, I, lane, 32);
            stage_planes(tslot, kNrm119, tf, M, lane, 32);
        }
        __syncwarp();
        u32 result = SR_DIS_ERR;
        s32 end = kAlignInf;
        if (walks) {
            end = align_dp(I, M, r, uslot, tslot, want_path ? choice : nullptr, lane);
            if (end < kAlignInf) result = (u32)end / (u32)(I + M);
        }
        int L = 0;
        if (want_path && result != SR_DIS_ERR) {
            __syncwarp();                                            // every lane's choice bytes are in shared memory
            if (lane == 0) {
                int i = I - 1, j = M - 1;
                for (;;) {
                    pbuf[L++] = (u16)(i | (j << 8));
                    if ((i == 0 && j == 0) || L == kPathMax) break;
                    const u32 ch = (choice[i * 32 + (j >> 2)] >> ((j & 3) * 2)) & 3u;
                    if (ch != 2u) --j;                               // diagonal or (i, j-1)
                    if (ch != 1u) --i;                               // diagonal or (i-1, j)
                }
            }
            L = __shfl_sync(0xFFFFFFFFu, L, 0);
            __syncwarp();
        }
        if (path) {
            u16 *dst = reinterpret_cast<u16 *>(path + (size_t)pr.out * kPathMax * 2);
            for (int q = lane; q < kPathMax; q += 32) dst[q] = q < L ? pbuf[L - 1 - q] : (u16)0xFFFFu;
        }
        if (lane == 0) {
            if (path_len) path_len[pr.out] = (u32)L;
            if (dis) dis[pr.out] = result;
        }
        if (pick_S && pr.in == pr.tpl * K + anchor) {                // C_0 = the anchor's features
            const u32 *src = reinterpret_cast<const u32 *>(uf);
            u32 *dst = reinterpret_cast<u32 *>(tpl_out + (size_t)pr.tpl * kFtrBytes);
            for (int w = lane; w < kFtrWords; w += 32) dst[w] = src[w];
            if (lane == 0 && anchor_out) anchor_out[pr.tpl] = anchor;
        }
    }
}

// One DBA update of every group with members: member l of group g (bank slot g*K + l) was aligned to C = tpl[g] with
// path pair index g*K + l; sum[j] += a_l[i] and cnt[j] += 1 for every point (i, j) of its path, then C[j] = sum[j] / cnt[j]
// (C division, truncating toward zero). C keeps its frame count; a group none of whose members aligned keeps C.
__global__ void __launch_bounds__(256)
average_update_kernel(const unsigned char *__restrict__ bank, u32 slot_stride, u32 K, const u32 *__restrict__ mask,
                      const u8 *__restrict__ path, const u32 *__restrict__ path_len, unsigned char *__restrict__ tpl) {
    __shared__ s32 sum[kMaxFrm * 12];
    __shared__ u32 cnt[kMaxFrm];
    const u32 g = blockIdx.x, m = mask[g];
    if (!m) return;
    for (int t = threadIdx.x; t < (int)kMaxFrm * 12; t += blockDim.x) sum[t] = 0;
    for (int t = threadIdx.x; t < (int)kMaxFrm; t += blockDim.x) cnt[t] = 0;
    __syncthreads();
    for (u32 l = 0; l < K; ++l) {
        if (!((m >> l) & 1u)) continue;
        const size_t s = (size_t)g * K + l;
        const int L = (int)path_len[s];
        const u16 *pp = reinterpret_cast<const u16 *>(path + s * kPathMax * 2);
        const s16 *a = reinterpret_cast<const s16 *>(bank + s * slot_stride + 4);
        for (int t = threadIdx.x; t < L * 12; t += blockDim.x) {
            const int q = t / 12, cf = t - q * 12;
            const u32 pt = pp[q], i = pt & 0xFFu, j = pt >> 8;
            atomicAdd(&sum[j * 12 + cf], (s32)a[i * 12 + cf]);
            if (cf == 0) atomicAdd(&cnt[j], 1u);
        }
    }
    __syncthreads();
    unsigned char *c = tpl + (size_t)g * kFtrBytes;
    const int M = (int)*reinterpret_cast<const u16 *>(c + 2);
    s16 *rows = reinterpret_cast<s16 *>(c + 4);
    for (int t = threadIdx.x; t < M * 12; t += blockDim.x) {
        const u32 n = cnt[t / 12];
        if (n) rows[t] = (s16)(sum[t] / (s32)n);
    }
}

// n pairs at radius band_r >= 0 (clamped to 118: every larger r is the full matrix)
cudaError_t launch_dtw_align(const void *in_base, u32 in_stride, const void *tpl_base, u32 tpl_stride, const void *pairs,
                             u32 n, int band_r, u8 *path, u32 *path_len, u32 *dis, const u32 *pick_S, const u32 *mask, u32 K,
                             void *tpl_out, u32 *anchor_out, int num_sms, cudaStream_t st) {
    if (n == 0) return cudaSuccess;
    if (band_r < 0) return cudaErrorInvalidValue;
    const int r = min(band_r, (int)kMaxFrm - 1);
    const size_t smem = (size_t)kAlignWarps * kAlignWarpBytes;
    cudaError_t e = cudaFuncSetAttribute(dtw_align_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
    const u32 grid = min((n + kAlignWarps - 1) / kAlignWarps, (u32)num_sms * 2u);   // two resident CTAs per SM
    dtw_align_kernel<<<grid, kAlignWarps * 32, smem, st>>>(
        static_cast<const unsigned char *>(in_base), in_stride, static_cast<const unsigned char *>(tpl_base), tpl_stride,
        static_cast<const AlignPair *>(pairs), n, r, path, path_len, dis, pick_S, mask, K,
        static_cast<unsigned char *>(tpl_out), anchor_out);
    return cudaGetLastError();
}

cudaError_t launch_average_update(const void *bank, u32 slot_stride, u32 K, u32 G, const u32 *mask, const u8 *path,
                                  const u32 *path_len, void *tpl, cudaStream_t st) {
    if (G == 0) return cudaSuccess;
    average_update_kernel<<<G, 256, 0, st>>>(static_cast<const unsigned char *>(bank), slot_stride, K, mask, path, path_len,
                                             static_cast<unsigned char *>(tpl));
    return cudaGetLastError();
}

}  // namespace srk
