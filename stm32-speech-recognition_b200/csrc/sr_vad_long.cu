// sr_vad_long.cu -- long-form VAD and per-segment recognition (include/sr_long.h): noise_atap (VAD.C:22-71) and the
// loop of VAD.C:97-218 with max_vc_con removed, over recordings of up to 2^27 samples, then spch_recg's decision
// (main.c:276-295) on every segment. Built on the batch kernel's pieces (sr_vad_core.cuh):
//   * K11a noise_atap: one warp per recording over its first n_len samples (noise_atap_warp);
//   * K11b block pass: the 80-sample block summaries (block_pass) of every recording, in work items of 32 blocks spread
//     over the whole grid rather than one warp per recording, so one 30-minute recording fills the GPU as well as a
//     batch of short ones. Each warp streams its items through two shared-memory buffers with bulk async copies
//     (chunk_issue): PCM is read once (2 B per sample) and 8 B per block are written to a workspace;
//   * K12 segment pass: one warp per recording walks windows of 1024 frames (vad_window): frames_pass over the summaries,
//     its `cin` (the carried last_sig) handed from pass to pass and window to window, then the endpoint FSM on the
//     window's activity bitmap (long_fsm_window), with the FSM's state (open or closed, and the length of the run that
//     crosses the window edge) carried into the next window and any number of segments emitted;
//   * recognition: a prefix sum over min(n_segs, max_segs) flattens the segments into one table (segment, PCM row,
//     atap), and the unchanged get_mfcc, template-scan and argmin kernels run on it with the segment count read from
//     device memory; a scatter writes one record per segment. No host round trip between VAD and recognition.
#include "sr_internal.h"
#include "../../include/sr_long.h"
#include "sr_vad_core.cuh"
#include "sr_dtw_core.cuh"

namespace srk {

__device__ __forceinline__ u32 rec_len(const u32 *lens, u32 b, u32 U) { return lens ? min(lens[b], U) : U; }

// ---- K11a: noise_atap over the first n_len samples; atap[b] untouched when n_len % 240 != 0 or n_len > lens[b] -------
constexpr int kLongWarps = 8;

__global__ void __launch_bounds__(kLongWarps * 32)
long_atap_kernel(const u16 *__restrict__ pcm, u32 U, u32 B, const u32 *__restrict__ lens, u32 n_len, atap_tag *__restrict__ atap) {
    const int lane = threadIdx.x & 31;
    const u32 b = blockIdx.x * kLongWarps + (threadIdx.x >> 5);
    if (b >= B || n_len == 0 || n_len % 240u != 0 || n_len > rec_len(lens, b, U)) return;   // VAD.C:33-36
    const u16 *x = pcm + (size_t)b * U;
    atap_tag at;
    noise_atap_warp(x, (reinterpret_cast<uintptr_t>(x) & 15) == 0, n_len, lane, at);
    if (lane == 0) atap[b] = at;
}

// ---- K11b: block summaries -------------------------------------------------------------------------------------------
// Work item i = chunk i % cpr of recording i / cpr: blocks [32c, 32c + 32) of it, those below its block count. Items are
// strided over the grid's warps (consecutive warps take consecutive chunks); items past a recording's end are skipped.
constexpr u32 kLongChunk = 32 * 80;
constexpr u32 kLongBuf = kLongChunk * 2 + 32;                    // one chunk + alignment slack (16-byte multiple)

__global__ void __launch_bounds__(kLongWarps * 32)
long_block_kernel(const u16 *__restrict__ pcm, u32 U, u32 B, const u32 *__restrict__ lens, const atap_tag *__restrict__ atap,
                  u32 *__restrict__ info, u32 info_stride, u32 cpr) {
    extern __shared__ __align__(128) unsigned char smem_raw[];
    __shared__ u64 bars[kLongWarps][2];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    unsigned char *buf0 = smem_raw + (size_t)warp * 2 * kLongBuf;               // buffer s at buf0 + s * kLongBuf
    if (lane == 0) { mbar_init(&bars[warp][0], 1); mbar_init(&bars[warp][1], 1); }
    if (threadIdx.x == 0) mbar_fence_init();
    __syncthreads();

    const size_t total_bytes = (size_t)B * U * 2;
    const bool base_aligned = (reinterpret_cast<uintptr_t>(pcm) & 15) == 0;
    const u64 n_items = (u64)B * cpr, stride = (u64)gridDim.x * kLongWarps;
    // recording, first block and block count of item i (0 blocks: the item lies past its recording's end)
    auto item = [&](u64 i, u32 &b, u32 &blk0, u32 &nb) {
        b = (u32)(i / cpr);
        blk0 = (u32)(i % cpr) * 32u;
        const u32 nfr = frames_of(rec_len(lens, b, U)), nblk = nfr ? nfr + 1 : 0;   // frame k = blocks k, k+1
        nb = blk0 < nblk ? min(32u, nblk - blk0) : 0u;
    };
    auto next_item = [&](u64 i, u32 &b, u32 &blk0, u32 &nb) {
        for (; i < n_items; i += stride) { item(i, b, blk0, nb); if (nb) break; }
        return i;
    };
    u32 b, blk0, nb, ph0 = 0, ph1 = 0;                                       // completed phases per buffer
    int shift_cur = 0, shift_nxt = 0;
    u64 it = next_item((u64)blockIdx.x * kLongWarps + warp, b, blk0, nb);
    if (it < n_items)
        shift_cur = chunk_issue(buf0, pcm, total_bytes, base_aligned, (size_t)b * U + 80u * blk0, 80u * nb, &bars[warp][0], lane);
    for (u32 k = 0; it < n_items; ++k) {
        const int s = k & 1;
        if (s) { mbar_wait(&bars[warp][1], ph1 & 1u); ++ph1; } else { mbar_wait(&bars[warp][0], ph0 & 1u); ++ph0; }
        const u32 cb = b, cblk0 = blk0, cnb = nb;
        const u64 nx = next_item(it + stride, b, blk0, nb);                  // the next item -> the other buffer
        if (nx < n_items)
            shift_nxt = chunk_issue(buf0 + (s ^ 1) * kLongBuf, pcm, total_bytes, base_aligned, (size_t)b * U + 80u * blk0, 80u * nb,
                                    &bars[warp][s ^ 1], lane);
        const atap_tag at = atap[cb];
        const u32 mid = at.mid_val, a_thl = mid + at.n_thl, b_thl = mid - at.n_thl;    // VAD.C:112-113 (u32 wrap)
        const u16 *x = reinterpret_cast<const u16 *>(buf0 + s * kLongBuf) + shift_cur;
        block_pass([&](u32 i) { return x + 80u * i; }, cnb, (shift_cur & 1) == 0, (shift_cur & 7) == 0, mid, a_thl, b_thl,
                   info + (size_t)cb * info_stride + 2u * cblk0, lane);
        __syncwarp();                                                          // this buffer is re-staged one item later
        shift_cur = shift_nxt;
        it = nx;
    }
}

// ---- K12: segments ---------------------------------------------------------------------------------------------------
// the FSM's actions on a recording: segment k < max_segs is written to out[2k], out[2k+1] (end SR_SEG_NULL until it closes)
struct LongSegOut {
    u32 max_segs;
    u32 *out;
    __device__ __forceinline__ void open(int lane, u32 n, u32 frame) {        // VAD.C:178: start = i - 7*80, i the 8th active
        if (lane == 0 && n < max_segs) { out[2 * n] = 80u * frame; out[2 * n + 1] = SR_SEG_NULL; }
    }
    __device__ __forceinline__ void close(int lane, u32 n, u32 frame) {       // VAD.C:201: end = i - 11*80 + 160, i the 11th inactive
        if (lane == 0 && n < max_segs) out[2 * n + 1] = 80u * frame + 80u;
    }
};

__global__ void __launch_bounds__(kLongWarps * 32)
long_segment_kernel(u32 U, u32 B, const u32 *__restrict__ lens, const atap_tag *__restrict__ atap, const u32 *__restrict__ info,
                    u32 info_stride, u32 max_segs, u32 *__restrict__ n_segs, u32 *__restrict__ seg_off) {
    const int lane = threadIdx.x & 31;
    const u32 b = blockIdx.x * kLongWarps + (threadIdx.x >> 5);
    if (b >= B) return;
    const u32 nfr = frames_of(rec_len(lens, b, U));
    const atap_tag at = atap[b];
    const u32 *inf = info + (size_t)b * info_stride;
    u32 *out = seg_off + (size_t)b * max_segs * 2;
    LongFsm f{false, 0u, 0u};
    LongSegOut act{max_segs, out};
    u32 cin = 0;                                                   // class of the last out-of-band sample so far (last_sig)
    for (u32 base = 0; base < nfr; base += 1024u) vad_window(inf, 0u, base, min(1024u, nfr - base), lane, at, cin, f, act);
    if (lane == 0) n_segs[b] = f.n + (f.open ? 1u : 0u);           // + the segment still open (end SR_SEG_NULL)
}

// ---- recognition plumbing --------------------------------------------------------------------------------------------
// exclusive prefix sum of min(n_segs[b], max_segs) -> first[b]; the total -> *n_flat. One CTA of 1024 threads.
__global__ void __launch_bounds__(1024) long_prefix_kernel(const u32 *__restrict__ n_segs, u32 B, u32 max_segs,
                                                           u32 *__restrict__ first, u32 *__restrict__ n_flat) {
    __shared__ u32 wsum[32];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    u32 carry = 0;
    for (u32 t0 = 0; t0 < B; t0 += 1024u) {
        const u32 b = t0 + threadIdx.x;
        const u32 m = b < B ? min(n_segs[b], max_segs) : 0u;
        u32 inc = m;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) { const u32 up = __shfl_up_sync(0xFFFFFFFFu, inc, o); if (lane >= o) inc += up; }
        if (lane == 31) wsum[warp] = inc;
        __syncthreads();
        if (warp == 0) {
            u32 w = wsum[lane];
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) { const u32 up = __shfl_up_sync(0xFFFFFFFFu, w, o); if (lane >= o) w += up; }
            wsum[lane] = w;
        }
        __syncthreads();
        const u32 before = carry + (warp ? wsum[warp - 1] : 0u) + inc - m;
        if (b < B) first[b] = before;
        carry += wsum[31];
        __syncthreads();
    }
    if (threadIdx.x == 0) *n_flat = carry;
}

// flat segment f = first[b] + k for k < min(n_segs[b], max_segs): its offsets, PCM row, atap and record slot b*max_segs+k
__global__ void long_flatten_kernel(const u32 *__restrict__ n_segs, const u32 *__restrict__ first, const u32 *__restrict__ seg_off,
                                    const atap_tag *__restrict__ atap, u32 B, u32 max_segs, u32 *__restrict__ seg2,
                                    u32 *__restrict__ row, u32 *__restrict__ slot, atap_tag *__restrict__ atap_seg) {
    const u32 i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= B * max_segs) return;
    const u32 b = i / max_segs, k = i % max_segs;
    if (k >= min(n_segs[b], max_segs)) return;
    const u32 fi = first[b] + k;
    seg2[2 * (size_t)fi] = seg_off[2 * (size_t)i];
    seg2[2 * (size_t)fi + 1] = seg_off[2 * (size_t)i + 1];
    row[fi] = b;
    slot[fi] = i;
    atap_seg[fi] = atap[b];
}

// status per flat segment (main.c:261-274): never closed -> VAD_FAIL, 0 frames -> MFCC_FAIL
__global__ void long_status_kernel(const u32 *__restrict__ seg2, const unsigned char *__restrict__ ftr, const u32 *__restrict__ n_flat,
                                   u8 *__restrict__ status) {
    const u32 i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= *n_flat) return;
    const u32 frm = (*reinterpret_cast<const u32 *>(ftr + (size_t)i * kFtrBytes)) >> 16;
    status[i] = seg2[2 * (size_t)i + 1] == SR_SEG_NULL ? SR_ST_VAD_FAIL : frm == 0 ? SR_ST_MFCC_FAIL : SR_ST_OK;
}

// the decision (decide, under a decision rule when kRule) of every flat segment into its record
template <bool kRule>
__global__ void long_scatter_kernel(const u32 *__restrict__ seg2, const u32 *__restrict__ slot, const unsigned char *__restrict__ ftr,
                                    const u8 *__restrict__ status, const u64 *__restrict__ best, const u32 *__restrict__ n_flat,
                                    sr_long_seg *__restrict__ rec, Rule rl) {
    const u32 g = kRule ? rule_lanes(rl) : 1u;
    const u32 i = (blockIdx.x * blockDim.x + threadIdx.x) / g;
    if (i >= *n_flat) return;
    Decision d;
    if (!decide<kRule>(best, i, status[i], rl, g, d)) return;
    sr_long_seg r;
    r.start = seg2[2 * (size_t)i]; r.end = seg2[2 * (size_t)i + 1]; r.status = d.status;
    r.frm_num = (*reinterpret_cast<const u32 *>(ftr + (size_t)i * kFtrBytes)) >> 16;
    r.best_idx = d.idx; r.best_dis = d.dis; r.cmd = d.cmd;
    rec[slot[i]] = r;
}

// ---- launchers -------------------------------------------------------------------------------------------------------
u32 long_info_stride(u32 U) { return 2u * (U / 80u + 2u); }

cudaError_t launch_long_atap(const u16 *pcm, u32 U, u32 B, const u32 *lens, u32 n_len, atap_tag *atap, cudaStream_t st) {
    if (B == 0) return cudaSuccess;
    long_atap_kernel<<<(B + kLongWarps - 1) / kLongWarps, kLongWarps * 32, 0, st>>>(pcm, U, B, lens, n_len, atap);
    return cudaGetLastError();
}

u32 long_block_grid(u32 U, u32 B, int num_sms) {
    const u64 items = (u64)B * ((U / 80u + 1u + 31u) / 32u);
    const u64 cap = (u64)num_sms * 2u;                             // two CTAs of 8 warps per SM (82 KB of buffers each)
    const u64 need = (items + kLongWarps - 1) / kLongWarps;
    return (u32)(need < cap ? (need ? need : 1) : cap);
}

cudaError_t launch_long_blocks(const u16 *pcm, u32 U, u32 B, const u32 *lens, const atap_tag *atap, u32 *info, int num_sms,
                               cudaStream_t st) {
    if (B == 0) return cudaSuccess;
    const size_t smem = (size_t)kLongWarps * 2 * kLongBuf;
    cudaError_t e = cudaFuncSetAttribute(long_block_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
    const u32 cpr = (U / 80u + 1u + 31u) / 32u;                   // chunks per recording: its blocks never exceed U / 80 + 1
    long_block_kernel<<<long_block_grid(U, B, num_sms), kLongWarps * 32, smem, st>>>(pcm, U, B, lens, atap, info,
                                                                                     long_info_stride(U), cpr);
    return cudaGetLastError();
}

cudaError_t launch_long_segments(u32 U, u32 B, const u32 *lens, const atap_tag *atap, const u32 *info, u32 max_segs, u32 *n_segs,
                                 u32 *seg_off, cudaStream_t st) {
    if (B == 0) return cudaSuccess;
    long_segment_kernel<<<(B + kLongWarps - 1) / kLongWarps, kLongWarps * 32, 0, st>>>(U, B, lens, atap, info, long_info_stride(U),
                                                                                     max_segs, n_segs, seg_off);
    return cudaGetLastError();
}

cudaError_t launch_long_flatten(const u32 *n_segs, const u32 *seg_off, const atap_tag *atap, u32 B, u32 max_segs, u32 *first,
                                u32 *n_flat, u32 *seg2, u32 *row, u32 *slot, atap_tag *atap_seg, cudaStream_t st, int step) {
    if (step == 0) {
        long_prefix_kernel<<<1, 1024, 0, st>>>(n_segs, B, max_segs, first, n_flat);
    } else {
        const u32 M = B * max_segs;
        long_flatten_kernel<<<(M + 255) / 256, 256, 0, st>>>(n_segs, first, seg_off, atap, B, max_segs, seg2, row, slot, atap_seg);
    }
    return cudaGetLastError();
}

cudaError_t launch_long_status(const u32 *seg2, const void *ftr, const u32 *n_flat, u32 M, u8 *status, cudaStream_t st) {
    long_status_kernel<<<(M + 255) / 256, 256, 0, st>>>(seg2, static_cast<const unsigned char *>(ftr), n_flat, status);
    return cudaGetLastError();
}

cudaError_t launch_long_scatter(const u32 *seg2, const u32 *slot, const void *ftr, const u8 *status, const u64 *best,
                                const u32 *n_flat, u32 M, sr_long_seg *rec, const Rule &rl, cudaStream_t st) {
    (rl.C ? long_scatter_kernel<true> : long_scatter_kernel<false>)<<<rule_grid(M, rl), 256, 0, st>>>(
        seg2, slot, static_cast<const unsigned char *>(ftr), status, best, n_flat, rec, rl);
    return cudaGetLastError();
}

}  // namespace srk
