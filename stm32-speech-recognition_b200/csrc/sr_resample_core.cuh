// sr_resample_core.cuh -- the polyphase resampler's rule in one place (DESIGN.md section 8), for K15's whole recordings
// (sr_resample.cu) and for K14's live streams at a rate (sr_long_stream.cu):
//   * output n reads phase (n*M + c) % L of the rate's [L][K] table against the input samples j = (n*M + c) / L, j - 1,
//     ..., j - K + 1 as centred s16 (resample_centre), and its exact s32 sum becomes a code by resample_code;
//   * the first n inputs fully support resample_ready(n) outputs: those whose newest sample (n*M + c) / L is below n.
// The tables live in sr_resample.cu, which holds the rates' taps; the other files reach them through resample_rate.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

// a rate of SR_RESAMPLE_RATES: (L, M) = (8000, rate) / gcd, K taps per phase, centre c = (N - 1) / 2
struct ResampleRate {
    uint32_t rate, L, M, K, c;
};

// the geometry of `rate`; false when it is not in SR_RESAMPLE_RATES
bool resample_rate(uint32_t rate, ResampleRate *out);
// the [L][K] phase table of `rate` (zero-padded to K taps per phase) on device dev, built on first use for every rate at
// once; NULL when the rate is unknown or the table could not be built
const int32_t *resample_phases(uint32_t rate, int dev);
// K15 (sr_resample_adc12_dev) on B recordings of device dev as one launch on st, for callers that have checked the rate,
// U_in, U_out and the pointers: the public call, and the host-buffer long-form calls at a rate under SR_LAUNCH
cudaError_t launch_resample_adc12(const uint16_t *in, uint32_t U_in, uint32_t B, const uint32_t *lens, uint32_t rate,
                                  uint16_t *out, uint32_t U_out, uint32_t *out_lens, int dev, cudaStream_t st);

// an input code as the tables' sums take it
__device__ __forceinline__ int16_t resample_centre(uint16_t x) { return (int16_t)((int32_t)x - 2048); }

// an output's s32 sum to its 12-bit code: round half up at 2^15, back to mid-code, clamp
__device__ __forceinline__ uint16_t resample_code(int32_t acc) {
    const int32_t y = 2048 + (int32_t)(((int64_t)acc + (1 << 14)) >> 15);
    return (uint16_t)(y < 0 ? 0 : (y > 4095 ? 4095 : y));
}

// n8(n) = max(0, ceil((n*L - c) / M)): the outputs whose every input sample is among the first n
__host__ __device__ __forceinline__ uint64_t resample_ready(uint64_t n, uint32_t L, uint32_t M, uint32_t c) {
    return n * L > c ? (n * L - c + M - 1) / M : 0;
}
