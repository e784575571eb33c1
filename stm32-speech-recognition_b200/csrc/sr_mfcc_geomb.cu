// sr_mfcc_geomb.cu -- get_mfcc (Src/Speech_Recog/MFCC.C:86-191) in the GEOM_B geometry of BASELINE configs[0]:
// 25 ms frames (200 samples), 10 ms hop (80), 256-point FFT, 128 spectral bins, 24 filters, 12 coefficients.
//
// EXTENSION, PARITY UNPINNED: the reference only implements 160/80/1024 (VAD.H:5-8, MFCC.H:8) and ships no 256-point
// FFT. What is built here is the reference's algorithm with the two sizes changed: the Hamming / Mel tables come from the
// reference's own Matlab formulas evaluated for frame_len = 200 and fft_point = 256 (tools/gen_tables.py;
// Matlab/matlab仿真/speech_recog.m:217-313), the FFT is the radix-4 routine of cr4_fft_1024_stm32.s:95-281 with three
// twiddled passes instead of four (the twiddle table is cumulative: its first 84 triples serve N = 256), and every
// integer rule of MFCC.C (pre-emphasis 95/100, hamm/1000, sqrtf*10, u32 energies, tri/100, log*100, DCT/100 into an
// s16) is kept. Its checker is oracle/sr_oracle.c::sro_mfcc_geom_b, whose FFT and tables tests/test_extension_refs.py
// holds to the exact DFT and to the tables' float64 formulas.
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
        // xs[-1] is read (MFCC.C:119). For start == 0 it is not a sample of the utterance (the previous row's last sample,
        // or before the batch): pinned to mid, as in the reference geometry's kernel (sr_mfcc.cu, stage_utterance)
        const u16 *xs = pcm + row * U + st;
        const bool at_origin = (st == 0);
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

// ---- test hook: the shared core's fft_radix4<N> alone, on n packed (re | im << 16) N-point inputs, one frame per warp.
// At N = 256 it is the only way to drive the GEOM_B FFT with complex, full-length input (the front end feeds it real,
// windowed 200-sample frames). Not part of recognition.
template <int N>
__global__ void __launch_bounds__(128)
fft_raw_n_kernel(const u32 *__restrict__ in, u32 n, u32 *__restrict__ out, const DevTables *__restrict__ tab) {
    __shared__ u32 xs[4][N];
    __shared__ u32 ys[4][N];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const u32 fr = blockIdx.x * 4 + warp;
    if (fr >= n) return;
    u32 *x = xs[warp], *y = ys[warp];
    for (int i = lane; i < N; i += 32) x[i] = in[(size_t)fr * N + i];
    __syncwarp();
    fft_radix4<N>(x, y, tab, lane);
    for (int i = lane; i < N; i += 32) out[(size_t)fr * N + i] = y[i];
}

cudaError_t launch_fft_raw_n(const u32 *in, u32 N, u32 n, u32 *out, cudaStream_t st) {
    if (n == 0) return cudaSuccess;
    const DevTables *tab = dev_tables();
    if (!tab) return cudaErrorInitializationError;
    const u32 grid = (n + 3) / 4;
    if (N == 256) fft_raw_n_kernel<256><<<grid, 128, 0, st>>>(in, n, out, tab);
    else if (N == 1024) fft_raw_n_kernel<1024><<<grid, 128, 0, st>>>(in, n, out, tab);
    else return cudaErrorInvalidValue;
    return cudaGetLastError();
}

// ---- test hooks: whole-domain checks of the float estimates under the MFCC kernels' exact integer steps. Each thread
// counts its mismatches over a grid-strided range; the device code is the kernels' own inline functions.
// log100 (float estimate + two correction loops) against the last L with thr[L] <= v, found by binary search, for v in
// [lo, hi), hi <= 2^32
__global__ void log100_check_kernel(u64 lo, u64 hi, const DevTables *__restrict__ tab, unsigned long long *bad) {
    unsigned long long n = 0;
    for (u64 i = lo + blockIdx.x * (u64)blockDim.x + threadIdx.x; i < hi; i += (u64)gridDim.x * blockDim.x) {
        const u32 v = (u32)i;
        int L = 0;
        if (v != 0) {
            int a = 0, b = 2218;                          // thr[a] <= v < thr[b + 1] (thr[2219] = 2^32 - 1 bounds nothing)
            while (a < b) {
                const int m = (a + b + 1) >> 1;
                if (tab->log_thr[m] <= v) a = m;
                else b = m - 1;
            }
            L = a;
        }
        if (log100(v, tab->log_thr) != (u32)L) ++n;
    }
    if (n) atomicAdd(bad, n);
}

// mag10_small over every (re, im) with |re|, |im| <= 8209 (which = 0; index i = (re + 8209) * 16419 + im + 8209, i <
// 16419^2), or mag10 over every s16 pair (which = 1; re = low half of i, im = high half, i < 2^32), against
// (u32)(sqrtf((float)pw) * 10) with pw = re^2 + im^2 as an s32: every step IEEE round-to-nearest, 0 for pw <= 0
__global__ void mag10_check_kernel(int which, u64 lo, u64 hi, unsigned long long *bad) {
    unsigned long long n = 0;
    for (u64 i = lo + blockIdx.x * (u64)blockDim.x + threadIdx.x; i < hi; i += (u64)gridDim.x * blockDim.x) {
        s32 re, im;
        if (which == 0) { re = (s32)(i / 16419) - 8209; im = (s32)(i % 16419) - 8209; }
        else { re = (s32)(s16)(u16)i; im = (s32)(s16)(u16)(i >> 16); }
        const s32 pw = (s32)(u32)((long long)re * re + (long long)im * im);
        const u32 want = pw <= 0 ? 0u : __float2uint_rz(__fmul_rn(__fsqrt_rn(__int2float_rn(pw)), 10.0f));
        const u32 got = which == 0 ? mag10_small((u32)re, (u32)im) : mag10((u32)re, (u32)im);
        if (got != want) ++n;
    }
    if (n) atomicAdd(bad, n);
}

cudaError_t launch_log100_check(u64 lo, u64 hi, unsigned long long *bad_dev, cudaStream_t st) {
    const DevTables *tab = dev_tables();
    if (!tab) return cudaErrorInitializationError;
    log100_check_kernel<<<132 * 8, 256, 0, st>>>(lo, hi, tab, bad_dev);
    return cudaGetLastError();
}

cudaError_t launch_mag10_check(int which, u64 lo, u64 hi, unsigned long long *bad_dev, cudaStream_t st) {
    mag10_check_kernel<<<132 * 8, 256, 0, st>>>(which, lo, hi, bad_dev);
    return cudaGetLastError();
}

}  // namespace srk
