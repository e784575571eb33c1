// sr_mfcc_core.cuh -- the integer rules of get_mfcc (Src/Speech_Recog/MFCC.C:86-191) and the radix-4 FFT of
// cr4_fft_1024_stm32.s:95-281, shared by the batch MFCC kernels and the drop-in fft (sr_mfcc.cu) and the GEOM_B
// extension (sr_mfcc_geomb.cu): the frame count, the pre-emphasis + Hamming term, the in-shared-memory FFT, the log
// lookup and the DCT epilogue.
#pragma once
#include "sr_common.cuh"

namespace srk {

// frame count of a segment, MFCC.C:102-107 (u32 wrap, u16 truncation); 0 = rejected / empty
template <u32 kFrameLen>
__device__ __forceinline__ int mfcc_frames(u32 start, u32 end, u32 U) {
    if (start == SR_SEG_NULL || end == SR_SEG_NULL || end > U || start > end) return 0;
    u32 len = end - start;
    if (len < kFrameLen) return 0;                // loop MFCC.C:113 never runs
    u32 n = (len - kFrameLen) / SR_FRAME_MOV + 1u;
    return n > SR_VV_FRM_MAX ? 0 : (int)n;
}

// pre-emphasis + Hamming of one sample, MFCC.C:115-124: cur = vc_dat[i], prv = vc_dat[i-1], hamm = the window weight;
// returns the s16-truncated value
__device__ __forceinline__ s32 preemph_hamm(u32 cur, u32 prv, u32 mid, u32 hamm) {
    const s32 c = (s32)(cur - mid), p = (s32)(prv - mid);
    const s32 t = (s32)((u32)c - (u32)((s32)((u32)p * 95u) / 100));
    return (s32)(s16)((s32)((u32)t * hamm) / 1000);
}

// The FFT of cr4_fft_1024_stm32.s for N = 256 or 1024 points, one warp, in shared memory: x holds the input in natural
// order, packed re | im << 16; y receives the output in bin order, same packing. A bit-reversed first pass of
// BUTFLY4ZERO_OPT (.s:132-178, 226-232), then the twiddled passes (.s:254-279) with strides 4 .. N/4; the twiddle table is
// cumulative, so its first 84 triples serve N = 256. Every store keeps the asm's STRH wrap (arbitrary complex input).
template <int N>
__device__ __forceinline__ void fft_radix4(const u32 *x, u32 *y, const DevTables *tab, int lane) {
    static_assert(N == 256 || N == 1024, "the twiddle table serves N = 256 and 1024");
    constexpr int kQ = N / 4, kRevShift = N == 256 ? 26 : 24;   // 32 - log2(N/4)
    for (int idx = lane; idx < kQ; idx += 32) {
        const int j = (int)(__brev((u32)idx) >> kRevShift);
        const u32 A = x[j], C = x[j + kQ], Bv = x[j + 2 * kQ], D = x[j + 3 * kQ];
        u32 o[8];
        cxadda4<0>(lo16s(A), hi16s(A), lo16s(Bv), hi16s(Bv), lo16s(C), hi16s(C), lo16s(D), hi16s(D),
                   o[0], o[1], o[2], o[3], o[4], o[5], o[6], o[7]);
#pragma unroll
        for (int m = 0; m < 4; ++m) y[4 * idx + m] = pack16(o[2 * m], o[2 * m + 1]);
    }
    __syncwarp();
    int toff = 0;
    for (int s = 4; s <= kQ; s <<= 2) {
        for (int t = lane; t < kQ; t += 32) {
            const int q = t % s, base = (t / s) * 4 * s;
            const int2 k3 = tab->tw[(toff + q) * 3], k2 = tab->tw[(toff + q) * 3 + 1], k1 = tab->tw[(toff + q) * 3 + 2];
            const u32 p0 = y[base + q], p1 = y[base + q + s], p2 = y[base + q + 2 * s], p3 = y[base + q + 3 * s];
            u32 Dr, Di, Cr, Ci, Br, Bi, o[8];
            cxmul(Dr, Di, lo16s(p3), hi16s(p3), (u32)k3.x, (u32)k3.y);
            cxmul(Cr, Ci, lo16s(p2), hi16s(p2), (u32)k2.x, (u32)k2.y);
            cxmul(Br, Bi, lo16s(p1), hi16s(p1), (u32)k1.x, (u32)k1.y);
            cxadda4<14>(lo16s(p0), hi16s(p0), Br, Bi, Cr, Ci, Dr, Di, o[0], o[1], o[2], o[3], o[4], o[5], o[6], o[7]);
#pragma unroll
            for (int m = 0; m < 4; ++m) y[base + q + m * s] = pack16(o[2 * m], o[2 * m + 1]);
        }
        __syncwarp();
        toff += s;
    }
}

// (u32)(log((double)v)*100) via the exact threshold table (MFCC.C:168; log(0) pinned to 0)
__device__ __forceinline__ u32 log100(u32 v, const u32 *thr) {
    if (v == 0) return 0;
    int L = (int)(__log2f(__uint2float_rn(v)) * 69.31471805599453f);
    L = max(0, min(L, 2218));
    while (v < thr[L]) --L;                       // thr[0] = 1 <= v, so this stops at L >= 0
    while (L < 2218 && v >= thr[L + 1]) ++L;
    return (u32)L;
}

// DCT, MFCC.C:173-183, from the warp's 24 log values lg: lane l < 24 sums half l & 1 of coefficient l >> 1 with its 12
// weights w, each term truncated toward zero; the halves meet by one shuffle and the coefficient is stored as s16 into
// the frame's output row. Lanes 24..31 compute a discarded copy.
__device__ __forceinline__ void dct_row(const u32 *lg, const s32 (&w)[12], unsigned char *row, int lane) {
    const u32 *lgp = lg + (lane & 1) * 12;
    s32 acc = 0;
#pragma unroll
    for (int i = 0; i < 12; ++i) acc += ((s32)lgp[i] * w[i]) / 100;
    acc += __shfl_xor_sync(0xFFFFFFFFu, acc, 1);
    if (lane < 24 && (lane & 1) == 0) *reinterpret_cast<s16 *>(row + (lane >> 1) * 2) = (s16)acc;
}

}  // namespace srk
