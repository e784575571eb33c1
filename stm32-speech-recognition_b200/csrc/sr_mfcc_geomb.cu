// sr_mfcc_geomb.cu -- get_mfcc (Src/Speech_Recog/MFCC.C:86-191) in the GEOM_B geometry of BASELINE configs[0]:
// 25 ms frames (200 samples), 10 ms hop (80), 256-point FFT, 128 spectral bins, 24 filters, 12 coefficients.
//
// EXTENSION, PARITY UNPINNED: the reference only implements 160/80/1024 (VAD.H:5-8, MFCC.H:8) and ships no 256-point
// FFT. What is built here is the reference's algorithm with the two sizes changed: the Hamming / Mel tables come from the
// reference's own Matlab formulas evaluated for frame_len = 200 and fft_point = 256 (tools/gen_tables.py;
// Matlab/matlab仿真/speech_recog.m:217-313), the FFT is the radix-4 routine of cr4_fft_1024_stm32.s:95-281 with three
// twiddled passes instead of four (the twiddle table is cumulative: its first 84 triples serve N = 256), and every
// integer rule of MFCC.C (pre-emphasis 95/100, hamm/1000, sqrtf*10, u32 energies, tri/100, log*100, DCT/100 into an
// s16) is kept. Its only checker is oracle/sr_oracle.c::sro_mfcc_geom_b.
//
// One CTA per utterance (persistent over the batch), one frame per warp. The FFT is the N = 256 instance of the shared
// core's fft_radix4 (sr_mfcc_core.cuh), the device code the drop-in fft runs at N = 1024 (s16 wrap on every store kept:
// a 200-sample frame does not enjoy the stage-0 collapse of the reference geometry). Not the benchmarked path: simple
// and exact rather than tuned.
#include "sr_mfcc_core.cuh"

namespace srk {

constexpr int kGbWarps = 8;
constexpr int kGbFrame = 200, kGbN = 256, kGbBins = 128;

__global__ void __launch_bounds__(kGbWarps * 32)
mfcc_geomb_kernel(const u16 *__restrict__ pcm, u32 U, u32 B, const u32 *__restrict__ seg, u32 seg_stride,
                  const atap_tag *__restrict__ atap, unsigned char *__restrict__ ftr, const DevTables *__restrict__ tab,
                  const u32 *__restrict__ row_map, const u32 *__restrict__ B_dev) {
    __shared__ u32 xin[kGbWarps][kGbN];
    __shared__ u32 ybuf[kGbWarps][kGbN];
    __shared__ u32 lg[kGbWarps][32];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (B_dev) B = min(B, *B_dev);
    u32 *x = xin[warp], *y = ybuf[warp];
    s32 dctk[12];
#pragma unroll
    for (int i = 0; i < 12; ++i) dctk[i] = (lane < 24) ? (s32)tab->dct[(lane >> 1) * 24 + (lane & 1) * 12 + i] : 0;
    int flo = 0, fhi = 0;
    if (lane < 24) { flo = tab->b_flt_lo[lane]; fhi = tab->b_flt_hi[lane]; }
    const u16 *tri = (lane & 1) ? tab->b_tri_odd : tab->b_tri_even;

    for (u32 b = blockIdx.x; b < B; b += gridDim.x) {
        const u32 st = seg[(size_t)b * seg_stride], en = seg[(size_t)b * seg_stride + 1];
        const s32 mid = (s32)atap[b].mid_val;
        const size_t row = row_map ? row_map[b] : b;
        const int F = mfcc_frames<kGbFrame>(st, en, U);
        if (threadIdx.x == 0) *reinterpret_cast<u16 *>(ftr + (size_t)b * kFtrBytes + 2) = (u16)F;
        const u16 *xs = pcm + row * U + st;                        // xs[-1] is read (MFCC.C:119); pinned to mid at the very start
        const bool at_origin = (row == 0 && st == 0);
        unsigned char *out_rows = ftr + (size_t)b * kFtrBytes + 4;
        for (int f = warp; f < F; f += kGbWarps) {
            const u16 *xf = xs + 80 * f;
            // pre-emphasis + Hamming, MFCC.C:115-124; zero padding to 256, MFCC.C:37-45
#pragma unroll
            for (int k = 0; k < 8; ++k) {
                const int i = lane + 32 * k;
                u32 v = 0;
                if (i < kGbFrame) {
                    const u32 p = (i == 0 && f == 0 && at_origin) ? (u32)mid : (u32)xf[i - 1];
                    v = (u32)(u16)preemph_hamm(xf[i], p, (u32)mid, tab->b_hamm[i]);
                }
                x[i] = v;
            }
            __syncwarp();
            fft_radix4<kGbN>(x, y, tab, lane);
            // magnitude (MFCC.C:49-60) and energy (MFCC.C:128-133) of bins 0..127 -> x[0..127]
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                const int i = lane + 32 * k;
                const u32 m = mag10(lo16s(y[i]), hi16s(y[i]));
                x[i] = m * m;
            }
            __syncwarp();
            // triangular filters (MFCC.C:136-162 with the GEOM_B centres), log (MFCC.C:165-170)
            {
                u32 acc = 0;
                for (int i = flo; i < fhi; ++i) acc += (x[i] * (u32)tri[i]) / 100u;
                lg[warp][lane] = (lane < 24) ? log100(acc, tab->log_thr) : 0u;
            }
            __syncwarp();
            dct_row(lg[warp], dctk, out_rows + (size_t)f * kRowBytes, lane);   // MFCC.C:173-183
            __syncwarp();
        }
    }
}

cudaError_t launch_mfcc_geomb(const u16 *pcm, u32 U, u32 B, const u32 *seg, u32 seg_stride, const atap_tag *atap, void *ftr,
                              int num_sms, cudaStream_t st, const u32 *row_map, const u32 *B_dev) {
    if (B == 0) return cudaSuccess;
    const DevTables *tab = dev_tables();
    if (!tab) return cudaErrorInitializationError;
    u32 grid = (u32)num_sms * 4u;
    if (grid > B) grid = B;
    mfcc_geomb_kernel<<<grid, kGbWarps * 32, 0, st>>>(pcm, U, B, seg, seg_stride, atap, static_cast<unsigned char *>(ftr), tab,
                                                     row_map, B_dev);
    return cudaGetLastError();
}

}  // namespace srk
