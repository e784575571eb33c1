// sr_vad.cu -- K0: batched noise_atap (Src/Speech_Recog/VAD.C:22-71) and VAD (VAD.C:97-218).
//
// One warp per utterance, persistent grid, utterances handed out dynamically (one atomic per utterance per warp, so CTAs
// that start late take fewer). A warp's utterances form one stream of 32-block chunks (2560 samples)
// through two shared-memory buffers: 1-D bulk async copies (TMA engine) keep the next chunk in flight while the
// current one is scanned, so HBM traffic is the algorithmic 2*U bytes per utterance.
// Each chunk runs the shared steps of sr_vad_core.cuh on the staged samples:
//   * noise_atap (noise_atap_warp): from the first staged chunk, three lanes per 240-sample block (IDP.2A sums, 16-byte
//     loads);
//   * VAD features (block_pass): frames overlap by 50 %, so the scan works on 80-sample BLOCKS (each sample is
//     touched once) and frame k = block k + block k+1. A block summary is a small monoid element:
//     sum |x-mid|, number of class alternations among its out-of-band samples, class of the last
//     out-of-band sample (the first one follows from the parity of the alternations). The band-
//     crossing count of the reference depends on `last_sig`, which is never reset between frames
//     (VAD.C:99): entering frame k it is the class of the last out-of-band sample at index <= i_k+78.
//     Only ONE pair per frame can see that carried-in state (the pair ending at the frame's first
//     out-of-band sample), so it is applied as a +1 correction; the carry itself is a warp scan.
//   * frames and endpoint FSM (vad_window, once per utterance from a fresh FSM state): 8 consecutive active frames open
//     a segment at the first of them, 11 consecutive inactive frames close it at the first of those -- evaluated with
//     bit tricks on the per-frame activity bitmap (one 32-frame word per lane) instead of a serial walk. The segments
//     are held in lanes (SegLanes): lane j < 6 is seg_off[j], so segments past the third are dropped without a branch.
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
    const u32 nfr = (do_vad && buf_len <= U) ? frames_of(buf_len) : 0;
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
            noise_atap_warp(pcm + ubase, false, n_len, lane, at);
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
            const u16 *x = reinterpret_cast<const u16 *>(buf) + shift;
            if (c0 == 0 && atap_staged) {
                noise_atap_warp(x, (shift & 7) == 0, n_len, lane, at);
                if (lane == 0) atap[b] = at;
                mid = at.mid_val; a_thl = mid + at.n_thl; b_thl = mid - at.n_thl;
            }
            const u32 blk0 = c0 / 80u;
            const u32 left = nblk > blk0 ? min(32u, nblk - blk0) : 0u;         // blocks of this chunk
            block_pass([&](u32 i) { return x + 80u * i; }, left, (shift & 1) == 0, (shift & 7) == 0, mid, a_thl, b_thl,
                       info + 2 * blk0, lane);
            __syncwarp();                                                      // this buffer is re-staged one chunk later
            shift_cur = shift_nxt;
        }

        // ---- VAD, VAD.C:97-218: frames from the block summaries ---------------------------------------------------
        if (do_vad) {
            u32 cin = 0;                                                       // last_sig before the first frame
            LongFsm f{false, 0u, 0u};
            SegLanes act{SR_SEG_NULL};
            vad_window(info, 0u, 0u, nfr, lane, at, cin, f, act);             // nfr <= 818: U <= 65535
            if (lane < 6) seg_off[(size_t)b * 6 + lane] = act.seg;
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
    const u32 max_frames = 2 * (frames_of(buf_len) + 2);                // 2 words per 80-sample block
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
