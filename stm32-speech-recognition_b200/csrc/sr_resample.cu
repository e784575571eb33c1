// sr_resample.cu -- K15: polyphase resampling of 12-bit codes to 8 kHz (sr_resample_adc12_dev, include/sr_synth.h).
//
// Output n reads phase p = (n*M + c) % L of the rate's table, h[p], h[p + L], ..., against the input samples
// j = (n*M + c) / L, j - 1, ... (DESIGN.md section 8). Outputs n and n + L read the same phase, M samples apart, so a
// CTA takes one tile of outputs of one recording, stages the input span the tile reads as centred s16 in shared
// memory, and hands out work items of one phase each: 32 lanes x R outputs L apart, so every lane of a warp reads the
// same tap (one uniform load from the phase table in global memory serves R multiply-adds per lane). All arithmetic is
// integer, and the tables keep |acc| < 2^31, so the s32 sums are exact. Results go through shared memory so that the
// stores to the output row are coalesced. The phase tables, the centring and the rounding are sr_resample_core.cuh's,
// shared with K14's live streams at a rate.
#include <cuda_runtime.h>
#include <stdint.h>
#include <algorithm>
#include <mutex>
#include <vector>
#include "../../include/sr_synth.h"
#include "sr_resample_core.cuh"
#include "sr_resample_taps.h"

namespace {

constexpr int kThreads = 512;
constexpr int kWarps = kThreads / 32;
constexpr int kRates = (int)(sizeof(sr_resample_rates) / sizeof(sr_resample_rates[0]));

// launch shape of one rate: tile = L * QB * 32 * R outputs, L * QB work items of 32 x R outputs
struct Plan {
    uint32_t L, M, K, c, R, QB, T, span;   // K taps per phase, span = staged samples per tile
    size_t smem;
};

Plan plan_of(const sr_resample_rate &r) {
    Plan p;
    p.L = r.L; p.M = r.M; p.K = (r.N + r.L - 1) / r.L; p.c = (r.N - 1) / 2;
    p.R = r.L == 1 ? 4 : 2;                  // L = 1: one phase, 16 items of 128 outputs; else one item per phase
    p.QB = r.L == 1 ? kWarps : 1;
    p.T = p.L * p.QB * 32u * p.R;
    // j_hi(n0 + T - 1) - j_hi(n0) <= ceil((T-1) M / L); K - 1 samples before j_hi(n0)
    p.span = (uint32_t)(((uint64_t)(p.T - 1) * p.M + p.L - 1) / p.L) + p.K;
    p.smem = ((size_t)p.span + p.T) * sizeof(int16_t);
    return p;
}

template <int R>
__global__ void __launch_bounds__(kThreads) resample_kernel(const uint16_t *__restrict__ in, uint32_t U_in,
                                                           const uint32_t *__restrict__ lens, uint16_t *__restrict__ out,
                                                           uint32_t U_out, uint32_t *__restrict__ out_lens,
                                                           const int32_t *__restrict__ hp, Plan p, uint32_t tiles) {
    extern __shared__ int16_t smem[];
    int16_t *s = smem;                                        // [span] centred input samples, 0 outside [0, len)
    uint16_t *o = reinterpret_cast<uint16_t *>(smem + p.span);   // [T] the tile's outputs
    const uint32_t b = blockIdx.x / tiles, tile = blockIdx.x % tiles;
    uint32_t len = lens ? lens[b] : U_in;
    if (len > U_in) len = U_in;
    const uint32_t olen = len ? (uint32_t)(((uint64_t)len * p.L + p.M - 1) / p.M) : 0u;
    if (tile == 0 && threadIdx.x == 0 && out_lens) out_lens[b] = olen;
    const uint64_t n0 = (uint64_t)tile * p.T;
    if (n0 >= olen) return;
    const uint32_t nt = (uint32_t)min((uint64_t)p.T, olen - n0);

    const int64_t jlo = (int64_t)((n0 * p.M + p.c) / p.L) - (int64_t)(p.K - 1);
    const uint16_t *x = in + (size_t)b * U_in;
    for (uint32_t i = threadIdx.x; i < p.span; i += kThreads) {
        const int64_t j = jlo + i;
        s[i] = (j >= 0 && j < (int64_t)len) ? resample_centre(__ldg(x + j)) : (int16_t)0;
    }
    __syncthreads();

    const uint32_t warp = threadIdx.x / 32, lane = threadIdx.x % 32;
    for (uint32_t item = warp; item < p.L * p.QB; item += kWarps) {
        const uint32_t ph0 = item % p.L, qb = item / p.L;
        // outputs n = n0 + q*L + ph0, q = qb*32R + lane + 32r: phase (t0 % L) and first sample (t0 / L) + q*M
        const uint64_t t0 = (n0 + ph0) * p.M + p.c;
        const int32_t *h = hp + (size_t)(t0 % p.L) * p.K;
        const int16_t *sb = s + (uint32_t)((int64_t)(t0 / p.L) - jlo) + (qb * 32u * R + lane) * p.M;
        int32_t acc[R];
#pragma unroll
        for (int r = 0; r < R; ++r) acc[r] = 0;
#pragma unroll 4
        for (uint32_t m = 0; m < p.K; ++m) {
            const int32_t tap = __ldg(h + m);
#pragma unroll
            for (int r = 0; r < R; ++r) acc[r] += tap * (int32_t)sb[(int32_t)(r * 32 * p.M) - (int32_t)m];
        }
#pragma unroll
        for (int r = 0; r < R; ++r) {
            const uint32_t nl = (qb * 32u * R + lane + 32u * r) * p.L + ph0;
            if (nl < nt) o[nl] = resample_code(acc[r]);
        }
    }
    __syncthreads();
    uint16_t *dst = out + (size_t)b * U_out + n0;
    for (uint32_t i = threadIdx.x; i < nt; i += kThreads) dst[i] = o[i];
}

bool usable(const void *ptr, int dev, unsigned align) {
    if (!ptr || ((uintptr_t)ptr & (align - 1))) return false;
    cudaPointerAttributes a;
    if (cudaPointerGetAttributes(&a, ptr) != cudaSuccess) {
        cudaGetLastError();
        return false;
    }
    return a.type == cudaMemoryTypeManaged || (a.type == cudaMemoryTypeDevice && a.device == dev);
}

}  // namespace

bool resample_rate(uint32_t rate, ResampleRate *out) {
    for (const sr_resample_rate &r : sr_resample_rates)
        if (r.rate == rate) {
            *out = {r.rate, r.L, r.M, (r.N + r.L - 1) / r.L, (r.N - 1) / 2};
            return true;
        }
    return false;
}

// per device: every rate's table as [L][K] phases (zero-padded to K taps) in one allocation
const int32_t *resample_phases(uint32_t rate, int dev) {
    static int32_t *tabs[64];
    static std::mutex mu;
    int k = 0;
    while (k < kRates && sr_resample_rates[k].rate != rate) ++k;
    if (k == kRates || dev < 0 || dev >= 64) return nullptr;
    std::lock_guard<std::mutex> lk(mu);
    size_t off[kRates], total = 0;
    for (int r = 0; r < kRates; ++r) {
        const sr_resample_rate &rr = sr_resample_rates[r];
        off[r] = total;
        total += (size_t)rr.L * ((rr.N + rr.L - 1) / rr.L);
    }
    if (!tabs[dev]) {
        std::vector<int32_t> all(total, 0);
        for (int r = 0; r < kRates; ++r) {
            const sr_resample_rate &rr = sr_resample_rates[r];
            const uint32_t K = (rr.N + rr.L - 1) / rr.L;
            for (uint32_t i = 0; i < rr.N; ++i) all[off[r] + (size_t)(i % rr.L) * K + i / rr.L] = rr.h[i];
        }
        int32_t *d = nullptr;
        if (cudaMalloc(&d, total * sizeof(int32_t)) != cudaSuccess) return nullptr;
        if (cudaMemcpy(d, all.data(), total * sizeof(int32_t), cudaMemcpyHostToDevice) != cudaSuccess) {
            cudaFree(d);
            return nullptr;
        }
        tabs[dev] = d;
    }
    return tabs[dev] + off[k];
}

// K15 on B recordings as one launch on st (declared in sr_resample_core.cuh); the caller has checked the rate, U_in, U_out,
// the grid (tiles * B < 2^31) and the pointers
cudaError_t launch_resample_adc12(const uint16_t *in, uint32_t U_in, uint32_t B, const uint32_t *lens, uint32_t rate,
                                  uint16_t *out, uint32_t U_out, uint32_t *out_lens, int dev, cudaStream_t st) {
    int k = 0;
    while (k < kRates && sr_resample_rates[k].rate != rate) ++k;
    if (k == kRates || dev < 0 || dev >= 64) return cudaErrorInvalidValue;
    const Plan p = plan_of(sr_resample_rates[k]);
    const uint64_t max_out = ((uint64_t)U_in * p.L + p.M - 1) / p.M;
    const uint64_t tiles = max_out ? (max_out + p.T - 1) / p.T : 1;
    // the kernels' shared memory limit raised, once per device, to what the largest tile needs
    static bool smem_set[64];
    static std::mutex mu;
    {
        std::lock_guard<std::mutex> lk(mu);
        if (!smem_set[dev]) {
            size_t smem_max = 0;
            for (const sr_resample_rate &rr : sr_resample_rates) smem_max = std::max(smem_max, plan_of(rr).smem);
            cudaError_t e = cudaFuncSetAttribute(resample_kernel<2>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_max);
            if (e == cudaSuccess)
                e = cudaFuncSetAttribute(resample_kernel<4>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_max);
            if (e != cudaSuccess) return e;
            smem_set[dev] = true;
        }
    }
    const int32_t *hp = resample_phases(rate, dev);
    if (!hp) return cudaErrorMemoryAllocation;
    const uint32_t grid = (uint32_t)(tiles * B);
    if (p.R == 4)
        resample_kernel<4><<<grid, kThreads, p.smem, st>>>(in, U_in, lens, out, U_out, out_lens, hp, p, (uint32_t)tiles);
    else
        resample_kernel<2><<<grid, kThreads, p.smem, st>>>(in, U_in, lens, out, U_out, out_lens, hp, p, (uint32_t)tiles);
    return cudaGetLastError();
}

extern "C" int sr_resample_adc12_dev(const uint16_t *in, uint32_t U_in, uint32_t B, const uint32_t *lens, uint32_t rate,
                                     uint16_t *out, uint32_t U_out, uint32_t *out_lens, void *cuda_stream) {
    int k = 0;
    while (k < kRates && sr_resample_rates[k].rate != rate) ++k;
    if (k == kRates || U_in > SR_RESAMPLE_U_MAX) return -1;
    const Plan p = plan_of(sr_resample_rates[k]);
    const uint64_t max_out = ((uint64_t)U_in * p.L + p.M - 1) / p.M;
    if ((uint64_t)U_out < max_out) return -1;
    if (B == 0) return 0;
    const uint64_t tiles = max_out ? (max_out + p.T - 1) / p.T : 1;
    if (tiles * B > 0x7FFFFFFFull) return -1;
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || dev >= 64) return -1;
    if (!usable(in, dev, 2) || !usable(out, dev, 2) || (lens && !usable(lens, dev, 4)) ||
        (out_lens && !usable(out_lens, dev, 4)))
        return -1;
    return launch_resample_adc12(in, U_in, B, lens, rate, out, U_out, out_lens, dev, static_cast<cudaStream_t>(cuda_stream)) ==
                   cudaSuccess
               ? 0
               : -1;
}
