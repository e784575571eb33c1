// sr_vad.cu -- K0: batched noise_atap (Src/Speech_Recog/VAD.C:22-71) and VAD (VAD.C:97-218).
//
// One warp per utterance, persistent grid, utterances handed out dynamically (one atomic per utterance per warp, so CTAs
// that start late take fewer). A warp's utterances form one stream of 32-block chunks (2560 samples)
// through two shared-memory buffers: 1-D bulk async copies (TMA engine) keep the next chunk in flight while the
// current one is scanned, so HBM traffic is the algorithmic 2*U bytes per utterance.
//   * noise_atap: from the first staged chunk, three lanes per 240-sample block (IDP.2A sums, 16-byte loads);
//   * VAD features: frames overlap by 50 %, so the scan works on 80-sample BLOCKS (each sample is
//     touched once) and frame k = block k + block k+1. A block summary is a small monoid element:
//     sum |x-mid|, number of class alternations among its out-of-band samples, class of the last
//     out-of-band sample (the first one follows from the parity of the alternations). The band-
//     crossing count of the reference depends on `last_sig`, which is never reset between frames
//     (VAD.C:99): entering frame k it is the class of the last out-of-band sample at index <= i_k+78.
//     Only ONE pair per frame can see that carried-in state (the pair ending at the frame's first
//     out-of-band sample), so it is applied as a +1 correction; the carry itself is a warp scan.
//   * endpoint FSM (VAD.C:164-216): 8 consecutive active frames open a segment at the first of
//     them, 11 consecutive inactive frames close it at the first of those -- evaluated with bit
//     tricks on the per-frame activity bitmap (one 32-frame word per lane) instead of a serial walk.
#include "sr_vad_core.cuh"

namespace srk {

constexpr int kVadMaxWarps = 20;

constexpr u32 kVadChunk = 32 * 80;                               // samples per staged chunk: one 80-sample block per lane

__global__ void __launch_bounds__(kVadMaxWarps * 32)
vad_kernel(const u16 *__restrict__ pcm, u32 U, u32 B, u32 n_len, u32 buf_len, int do_atap, int do_vad,
           atap_tag *__restrict__ atap, u32 *__restrict__ seg_off, u32 buf_bytes, u32 max_frames,
           u32 *__restrict__ work /* [0] next utterance to hand out, [1] warps finished; NULL: static striding */) {
    extern __shared__ __align__(128) unsigned char smem_raw[];
    __shared__ u64 bars[kVadMaxWarps][2];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nwarps = blockDim.x >> 5;
    unsigned char *buf0 = smem_raw + (size_t)warp * 2 * buf_bytes, *buf1 = buf0 + buf_bytes;   // double buffer
    u32 *info = reinterpret_cast<u32 *>(smem_raw + (size_t)nwarps * 2 * buf_bytes) + (size_t)warp * max_frames;
    if (lane == 0) { mbar_init(&bars[warp][0], 1); mbar_init(&bars[warp][1], 1); }
    if (threadIdx.x == 0) mbar_fence_init();
    __syncthreads();

    const size_t total_bytes = (size_t)B * U * 2;
    const bool base_aligned = (reinterpret_cast<uintptr_t>(pcm) & 15) == 0;

    // the same for every utterance of the launch
    const bool atap_on = do_atap && n_len != 0 && (n_len % 240u) == 0 && n_len <= U;   // VAD.C:33-36: else untouched
    // frames i = 0,80,.. while i < buf_len-160 (VAD.C:121); buf_len <= 160 reads past the buffer in the reference
    // (int -> u32 compare) -- here: no frames.
    const u32 nfr = (do_vad && buf_len > SR_FRAME_LEN && buf_len <= U) ? (buf_len - SR_FRAME_LEN + SR_FRAME_MOV - 1) / SR_FRAME_MOV : 0;
    const u32 nblk = nfr ? nfr + 1 : 0;                            // frame k = blocks k, k+1
    const u32 vad_samples = 80u * nblk;                            // <= buf_len
    const bool atap_staged = atap_on && n_len <= kVadChunk;        // noise_atap from the first staged chunk
    const u32 total = max(vad_samples, atap_staged ? n_len : 0u);  // samples staged per utterance

    // The warp's chunks (32 blocks each, utterance after utterance) form one stream through the two buffers: chunk k+1 is in
    // flight while chunk k is scanned, across utterance boundaries too. Every PCM byte is read from HBM once.
    // Utterances are handed out DYNAMICALLY (one atomic per utterance per warp): a CTA that starts late -- e.g. because a
    // collective of the previous batch still holds its SM -- simply takes fewer. With static striding every late CTA
    // delayed the whole kernel (measured: 0.27 -> 0.42 ms at 8 GPUs, where the score all-gather overlaps this kernel).
    const u32 stride = gridDim.x * nwarps;
    auto claim = [&]() -> u32 {
        u32 v = 0;
        if (lane == 0) v = atomicAdd(&work[0], 1u);
        return __shfl_sync(0xFFFFFFFFu, v, 0);
    };
    u32 b = work ? claim() : blockIdx.x * nwarps + warp;
    bool have_next = false;
    u32 b_next = 0;
    u32 k = 0, ph0 = 0, ph1 = 0;                                   // chunk counter, completed phases per buffer
    int shift_cur = 0, shift_nxt = 0;
    if (total && b < B)
        shift_cur = chunk_issue(buf0, pcm, total_bytes, base_aligned, (size_t)b * U, min(kVadChunk, total), &bars[warp][0], lane);

    while (b < B) {
        const size_t ubase = (size_t)b * U;
        atap_tag at = atap[b];

        // ---- noise_atap, VAD.C:22-71, when the window does not fit the first chunk: straight from global ------------
        if (atap_on && !atap_staged) {
            u32 m, max_sum, abs_sum;
            atap_stats(pcm + ubase, false, n_len, lane, m, max_sum, abs_sum);
            atap_finish(at, n_len, m, max_sum, abs_sum);
            if (lane == 0) atap[b] = at;
        }
        u32 mid = at.mid_val, a_thl = mid + at.n_thl, b_thl = mid - at.n_thl;            // VAD.C:112-113 (u32 wrap)

        for (u32 c0 = 0; c0 < total; c0 += kVadChunk, ++k) {
            const bool odd = k & 1u;
            unsigned char *buf = odd ? buf1 : buf0;
            if (odd) { mbar_wait(&bars[warp][1], ph1 & 1u); ++ph1; } else { mbar_wait(&bars[warp][0], ph0 & 1u); ++ph0; }
            {                                                                  // next chunk of the stream -> other buffer
                u32 nb = b, nc0 = c0 + kVadChunk;
                if (nc0 >= total) {                                            // first chunk of this warp's next utterance
                    if (!have_next) { b_next = work ? claim() : b + stride; have_next = true; }
                    nb = b_next; nc0 = 0;
                }
                if (nb < B)
                    shift_nxt = chunk_issue(odd ? buf0 : buf1, pcm, total_bytes, base_aligned, (size_t)nb * U + nc0,
                                            min(kVadChunk, total - nc0), &bars[warp][odd ? 0 : 1], lane);
            }
            const int shift = shift_cur;
            VadWarpView v;
            v.x = reinterpret_cast<const u16 *>(buf) + shift;
            v.vec_ok = (shift & 7) == 0;
            if (c0 == 0 && atap_staged) {
                u32 m, max_sum, abs_sum;
                atap_stats(v.x, v.vec_ok, n_len, lane, m, max_sum, abs_sum);   // VAD.C:41-63
                atap_finish(at, n_len, m, max_sum, abs_sum);
                if (lane == 0) atap[b] = at;
                mid = m; a_thl = mid + at.n_thl; b_thl = mid - at.n_thl;
            }
            const u32 blk0 = c0 / 80u;
            const u32 left = nblk > blk0 ? nblk - blk0 : 0u;                   // blocks of this chunk
            if (left <= 4u && (shift & 1) == 0) {                              // few blocks: eight lanes per block
                if (left) {
                    u32 bs, fl;
                    block_scan_split8(v.x, lane, left, mid, a_thl, b_thl, bs, fl);
                    const u32 blk = blk0 + (u32)(lane >> 3);
                    if ((lane & 7) == 0 && blk < nblk) { info[2 * blk] = bs; info[2 * blk + 1] = fl; }
                }
            } else if ((u32)lane < left) {
                const u32 blk = blk0 + (u32)lane;
                u32 bs, fl;
                block_scan(v, 80u * (u32)lane, mid, a_thl, b_thl, bs, fl);
                info[2 * blk] = bs; info[2 * blk + 1] = fl;
            }
            __syncwarp();                                                      // this buffer is re-staged one chunk later
            shift_cur = shift_nxt;
        }

        // ---- VAD, VAD.C:97-218: frames from the block summaries ---------------------------------------------------
        if (do_vad) {
            u32 seg[6] = {SR_SEG_NULL, SR_SEG_NULL, SR_SEG_NULL, SR_SEG_NULL, SR_SEG_NULL, SR_SEG_NULL};
            if (nfr > 0) {
                u32 aw = 0;                                                    // lane j: activity of frames 32j..32j+31
                u32 cin = 0;                                                   // class of last out-of-band sample before this pass
                for (u32 k0 = 0, j = 0; k0 < nfr; k0 += 32, ++j) {
                    const u32 word = frames_pass(info, k0, nfr, lane, at, cin);
                    if ((u32)lane == j) aw = word;
                }
                fsm_segments(aw, nfr, lane, seg);                             // endpoint FSM on the bitmap
            }
            if (lane < 6) {
                u32 val = seg[0];
#pragma unroll
                for (int j = 1; j < 6; ++j) if (lane == j) val = seg[j];
                seg_off[(size_t)b * 6 + lane] = val;
            }
        }
        __syncwarp();
        b = have_next ? b_next : (work ? claim() : b + stride);
        have_next = false;
    }
    // the last warp out re-arms the counters for the next launch on this stream
    if (work && lane == 0) {
        __threadfence();
        if (atomicAdd(&work[1], 1u) == gridDim.x * (u32)nwarps - 1u) { work[0] = 0; work[1] = 0; }
    }
}

cudaError_t launch_vad(const u16 *pcm, u32 U, u32 B, u32 n_len, u32 buf_len, int do_atap, int do_vad,
                       atap_tag *atap, u32 *seg_off, int num_sms, cudaStream_t st, u32 *work) {
    if (B == 0) return cudaSuccess;
    const u32 buf_bytes = kVadChunk * 2 + 32;                          // one 32-block chunk + alignment slack (16-byte multiple)
    const u32 max_frames = 2 * ((buf_len > 160 ? (buf_len - 160 + 79) / 80 : 0) + 2);   // 2 words per 80-sample block
    const size_t per_warp = 2 * (size_t)buf_bytes + (size_t)max_frames * 4;   // two chunk buffers + block summaries
    int warps = (int)((220 * 1024) / per_warp);
    if (warps < 1) return cudaErrorInvalidValue;
    if (warps > kVadMaxWarps) warps = kVadMaxWarps;
    const size_t smem = per_warp * warps;
    cudaError_t e = cudaFuncSetAttribute(vad_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 224 * 1024);   // + 96 B static barriers <= 227 KB
    if (e != cudaSuccess) return e;
    u32 grid = (B + warps - 1) / warps;
    size_t resident = (224 * 1024) / (smem + 2048);                     // CTAs that fit one SM (smem-limited)
    if (resident < 1) resident = 1;
    const u32 cap = (u32)num_sms * (u32)resident;                       // persistent: one wave, warps stride over utterances
    if (grid > cap) grid = cap;
    vad_kernel<<<grid, warps * 32, smem, st>>>(pcm, U, B, n_len, buf_len, do_atap, do_vad, atap, seg_off, buf_bytes,
                                              max_frames, work);
    return cudaGetLastError();
}

}  // namespace srk
