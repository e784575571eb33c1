// sr_vad_core.cuh -- one warp's noise_atap (VAD.C:22-71) and VAD (VAD.C:97-218), shared by the four VAD kernels: the
// batch kernel K0 (sr_vad.cu: samples staged in shared memory), the long-form kernels K11/K12 (sr_vad_long.cu: the same
// staging), the fixed-capture streams K4 (sr_stream.cu: samples read from the streams' device rows) and the live streams
// K14 (sr_long_stream.cu: samples in a ring). Each kernel runs the same three steps:
//   * noise_atap_warp: the thresholds from the calibration window;
//   * block_pass: the summaries of 80-sample blocks, wherever the caller keeps the samples;
//   * vad_window: up to 1 024 frames from those summaries (frames_pass, last_sig carried in `cin`), then the endpoint FSM
//     continued from its carried state (long_fsm_window); the caller's act says what an opening and a closing do.
#pragma once
#include "sr_common.cuh"

namespace srk {

// frames i = 80k while i < len - 160 (VAD.C:121); none for len <= 160 (the reference compares as u32 and reads past the
// buffer). Frame k = blocks k, k + 1.
__host__ __device__ __forceinline__ u32 frames_of(u32 len) {
    return len > SR_FRAME_LEN ? (len - SR_FRAME_LEN + SR_FRAME_MOV - 1) / SR_FRAME_MOV : 0u;
}

__device__ __forceinline__ u32 warp_sum(u32 v) {
#pragma unroll
    for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xFFFFFFFFu, v, o);
    return v;
}
__device__ __forceinline__ u32 warp_max(u32 v) {
#pragma unroll
    for (int o = 16; o; o >>= 1) v = max(v, __shfl_xor_sync(0xFFFFFFFFu, v, o));
    return v;
}

// noise_atap (VAD.C:22-71) over samples x[0, n_len), n_len % 240 == 0, into at. Its three sums (VAD.C:41-63): mid =
// sum/n_len, max_sum = sum over 240-sample blocks of max|x-mid|, abs_sum = sum |x-mid|. Vector form (x 16-byte aligned,
// n_len <= 2560): lane l owns samples [80l, 80l+80) (three lanes per 240-block), 16-byte loads, IDP.2A for the plain sum.
__device__ __forceinline__ void noise_atap_warp(const u16 *x, bool vec_ok, u32 n_len, int lane, atap_tag &at) {
    u32 mid, max_sum = 0, abs_sum = 0;
    if (vec_ok && n_len <= 2560u) {
        const bool act = 80u * (u32)lane < n_len;
        const uint4 *p = reinterpret_cast<const uint4 *>(x + (act ? 80 * lane : 0));
        u32 s = 0;
#pragma unroll
        for (int c = 0; c < 10; ++c) {
            const uint4 q = p[c];
            s = __dp2a_lo(q.x, 0x0101u, s); s = __dp2a_lo(q.y, 0x0101u, s);
            s = __dp2a_lo(q.z, 0x0101u, s); s = __dp2a_lo(q.w, 0x0101u, s);
        }
        mid = warp_sum(act ? s : 0u) / n_len;
        u32 mx = 0, sm = 0;
#pragma unroll
        for (int c = 0; c < 10; ++c) {
            const uint4 q = p[c];
            const u32 w[4] = {q.x, q.y, q.z, q.w};
#pragma unroll
            for (int k = 0; k < 8; ++k) {
                const u32 v = (k & 1) ? (w[k >> 1] >> 16) : (w[k >> 1] & 0xFFFFu);
                const u32 d = __usad(v, mid, 0u);
                mx = max(mx, d); sm += d;
            }
        }
        if (!act) { mx = 0; sm = 0; }
        const u32 m1 = __shfl_down_sync(0xFFFFFFFFu, mx, 1), m2 = __shfl_down_sync(0xFFFFFFFFu, mx, 2);
        const u32 bmax = (act && lane % 3 == 0) ? max(mx, max(m1, m2)) : 0u;      // lanes 3k..3k+2 = block k
        max_sum = warp_sum(bmax);
        abs_sum = warp_sum(sm);
    } else {
        u32 s = 0;
        for (u32 i = lane; i < n_len; i += 32) s += x[i];
        mid = warp_sum(s) / n_len;                                   // VAD.C:41-45
        for (u32 i = 0; i < n_len; i += 240u) {                      // VAD.C:48-63
            u32 mx = 0, sm = 0;
            for (u32 h = lane; h < 240u; h += 32) { const u32 v = x[i + h], a = v > mid ? v - mid : mid - v; mx = max(mx, a); sm += a; }
            max_sum += warp_max(mx);
            abs_sum += sm;
        }
        abs_sum = warp_sum(abs_sum);
    }
    abs_sum /= (n_len / SR_FRAME_LEN);                               // VAD.C:65
    max_sum /= (n_len / 240u);                                       // VAD.C:66
    at.mid_val = mid;
    at.n_thl = (u16)max_sum;                                         // n_thl_ratio 1, VAD.C:68
    at.s_thl = abs_sum * 11u / 10u;                                  // s_thl_ratio 11/10, VAD.C:69
    at.z_thl = 2;                                                    // 160*2/160/1, VAD.C:70
}

// per-block summary: bs = sum |x-mid| over the 80 samples; flags = zc (bits 0..6, alternations inside the
// block) | lc << 7 (class of last out-of-band sample, 0 none / 1 below / 2 above) | lcA << 9 (same over the
// first 79 samples) | p0 << 11 (sample 0 is out of band)
//
// flags of one 80-sample block from its bitmaps (H = ">= a_thl", L = "< b_thl", bit i = sample i; words 0..31, 32..63,
// 64..79). An alternation is an out-of-band sample ("marker", N = H|L) whose class differs from the previous marker's;
// the first marker of the block never counts here (the frame-level pass applies the carried-in state). "Previous
// marker is H" for every position comes from ONE 80-bit addition: in (H << 1) + ~N a carry injected just above each
// H marker ripples through the non-markers and lands on the next marker. Bit 80 of the sum says the last marker of the
// block is H; bit 79, xor-ed with ~N, says the same for the first 79 samples.
__device__ __forceinline__ u32 block_flags(u32 (&H)[3], u32 (&L)[3]) {
#pragma unroll
    for (int k = 0; k < 3; ++k) L[k] &= ~H[k];                              // ">= a" is tested first, "< b" only else
    const u32 n0 = ~(H[0] | L[0]), n1 = ~(H[1] | L[1]), n2 = ~(H[2] | L[2]) & 0xFFFFu;   // bit 80 acts as a marker
    u32 sh0, sh1, sh2, sl0, sl1, sl2;
    asm("{\n add.cc.u32 %0, %3, %6;\n addc.cc.u32 %1, %4, %7;\n addc.u32 %2, %5, %8;\n}"
        : "=r"(sh0), "=r"(sh1), "=r"(sh2)
        : "r"(H[0] << 1), "r"(__funnelshift_l(H[0], H[1], 1)), "r"(__funnelshift_l(H[1], H[2], 1)), "r"(n0), "r"(n1), "r"(n2));
    asm("{\n add.cc.u32 %0, %3, %6;\n addc.cc.u32 %1, %4, %7;\n addc.u32 %2, %5, %8;\n}"
        : "=r"(sl0), "=r"(sl1), "=r"(sl2)
        : "r"(L[0] << 1), "r"(__funnelshift_l(L[0], L[1], 1)), "r"(__funnelshift_l(L[1], L[2], 1)), "r"(n0), "r"(n1), "r"(n2));
    const u32 zc = __popc((L[0] & sh0) | (H[0] & sl0)) + __popc((L[1] & sh1) | (H[1] & sl1)) +
                   __popc((L[2] & sh2) | (H[2] & sl2));
    const u32 last = ((sh2 >> 15) & 2u) | ((sl2 >> 16) & 1u);               // bit 16 of word 2 = position 80
    const u32 lastA = (((sh2 ^ n2) >> 14) & 2u) | (((sl2 ^ n2) >> 15) & 1u); // position 79
    const u32 p0 = ~n0 & 1u;
    return zc | (last << 7) | (lastA << 9) | (p0 << 11);
}

// Per-block summary, built from bitmaps. Two samples per 32-bit word stay packed: |x-mid| = max - min per 16-bit lane
// (VIMNMX.U16x2), summed by IDP.2A; the band compares are carries of w + (0 - (t << 16)) (high sample) and
// (w << 16) + (0 - (t << 16)) (low sample, one LEA), shifted MSB-first into the bitmaps by IMAD.X (x*2 + carry, FMA pipe):
// per sample 3 ALU-pipe and 3 FMA-pipe instructions -- the ALU pipe is what bounds this kernel. t == 0 and t > 0xFFFF
// are patched after the loop; mid > 0xFFFF (only possible with a caller-supplied atap_tag) takes the plain loop.
// p = the block's first sample; vec_ok: p is 16-byte aligned (uint4 loads).
__device__ __forceinline__ void block_scan(const u16 *p, bool vec_ok, u32 mid, u32 a_thl, u32 b_thl, u32 &bs_out,
                                           u32 &flags_out) {
    u32 bs = 0;
    u32 H[3], L[3];
    if (mid <= 0xFFFFu) {
        u32 gA[3] = {0, 0, 0}, gB[3] = {0, 0, 0};      // "s >= a_thl", "s >= b_thl"; samples 0..31, 32..63, 64..79
        u32 bsx = 0, bsn = 0;
        const u32 mid2 = mid | (mid << 16), na = 0u - (a_thl << 16), nb = 0u - (b_thl << 16);
#pragma unroll
        for (int c = 0; c < 10; ++c) {
            u32 w[4];
            if (vec_ok) {
                const uint4 q = *reinterpret_cast<const uint4 *>(p + 8 * c);
                w[0] = q.x; w[1] = q.y; w[2] = q.z; w[3] = q.w;
            } else {
#pragma unroll
                for (int j = 0; j < 4; ++j) w[j] = (u32)p[8 * c + 2 * j] | ((u32)p[8 * c + 2 * j + 1] << 16);
            }
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                const int g = (8 * c + 2 * j) >> 5;
                u32 mn;
                asm("min.u16x2 %0, %1, %2;" : "=r"(mn) : "r"(w[j]), "r"(mid2));
                // VAD.C:126-129: |x-mid| = max - min = x + mid - 2 min(x, mid): one packed min (ALU pipe, the busy one) and two
                // IDP.2A sums (FMA pipe) per sample pair; the block total is assembled after the loop
                bsx = __dp2a_lo(w[j], 0x0101u, bsx);
                bsn = __dp2a_lo(mn, 0x0101u, bsn);
                asm("{\n .reg .u32 t, l;\n shl.b32 l, %2, 16;\n"
                    " add.cc.u32 t, l, %3;\n madc.lo.u32 %0, %0, 2, 0;\n"  // VAD.C:134-141 / 143-156, low sample
                    " add.cc.u32 t, l, %4;\n madc.lo.u32 %1, %1, 2, 0;\n"
                    " add.cc.u32 t, %2, %3;\n madc.lo.u32 %0, %0, 2, 0;\n" // high sample
                    " add.cc.u32 t, %2, %4;\n madc.lo.u32 %1, %1, 2, 0;\n}"
                    : "+r"(gA[g]), "+r"(gB[g])
                    : "r"(w[j]), "r"(na), "r"(nb));
            }
        }
        bs = bsx + 80u * mid - 2u * bsn;
        H[0] = __brev(gA[0]); H[1] = __brev(gA[1]); H[2] = __brev(gA[2]) >> 16;
        L[0] = ~__brev(gB[0]); L[1] = ~__brev(gB[1]); L[2] = ~(__brev(gB[2]) >> 16) & 0xFFFFu;
        if (a_thl == 0) { H[0] = 0xFFFFFFFFu; H[1] = 0xFFFFFFFFu; H[2] = 0xFFFFu; }   // s >= 0 always
        if (a_thl > 0xFFFFu) { H[0] = 0; H[1] = 0; H[2] = 0; }                         // s >= t never
        if (b_thl == 0) { L[0] = 0; L[1] = 0; L[2] = 0; }                              // s <  0 never
        if (b_thl > 0xFFFFu) { L[0] = 0xFFFFFFFFu; L[1] = 0xFFFFFFFFu; L[2] = 0xFFFFu; }   // s <  t always
    } else {
#pragma unroll
        for (int k = 0; k < 3; ++k) {
            u32 hw = 0, lw = 0;
            const int n = k < 2 ? 32 : 16;
#pragma unroll 1
            for (int i = 0; i < n; ++i) {
                const u32 s = p[32 * k + i];
                bs = __usad(s, mid, bs);
                hw |= (s >= a_thl ? 1u : 0u) << i;
                lw |= (s < b_thl ? 1u : 0u) << i;
            }
            H[k] = hw; L[k] = lw;
        }
    }
    bs_out = bs;
    flags_out = block_flags(H, L);
}

// The same summary for up to four blocks at once, eight lanes per block (ten samples each): used for the last pass of
// an utterance when only a few blocks remain, instead of a full 80-sample pass with most lanes idle. x must be
// 4-byte aligned. Every lane of a group returns the group's result; groups >= nblocks return garbage.
__device__ __forceinline__ void block_scan_split8(const u16 *x, int lane, u32 nblocks, u32 mid, u32 a_thl, u32 b_thl,
                                                  u32 &bs_out, u32 &flags_out) {
    const int g = lane >> 3, j = lane & 7;
    const bool act = (u32)g < nblocks;
    const u32 *pw = reinterpret_cast<const u32 *>(x + (act ? 80 * g + 10 * j : 0));
    const u32 na = 0u - a_thl, nb = 0u - b_thl;
    u32 bs = 0, gA = 0, gB = 0;
#pragma unroll
    for (int c = 0; c < 5; ++c) {
        const u32 w = pw[c];
#pragma unroll
        for (int k = 0; k < 2; ++k) {
            const u32 s = k ? (w >> 16) : (w & 0xFFFFu);
            bs = __usad(s, mid, bs);
            asm("{\n .reg .u32 t;\n"
                " add.cc.u32 t, %2, %3;\n madc.lo.u32 %0, %0, 2, 0;\n"
                " add.cc.u32 t, %2, %4;\n madc.lo.u32 %1, %1, 2, 0;\n}"
                : "+r"(gA), "+r"(gB)
                : "r"(s), "r"(na), "r"(nb));
        }
    }
    u32 h10 = __brev(gA) >> 22, l10 = ~(__brev(gB) >> 22) & 0x3FFu;       // sample i of this lane at bit i
    if (a_thl == 0) h10 = 0x3FFu;
    if (b_thl == 0) l10 = 0;
    // place the 10 bits at position 10*j of the 80-bit block bitmap, then OR / add over the group's 8 lanes
    const int pos = 10 * j;
    const u64 hv = pos < 64 ? ((u64)h10 << pos) : 0ull, lv = pos < 64 ? ((u64)l10 << pos) : 0ull;
    u32 H[3], L[3];
    H[0] = (u32)hv; H[1] = (u32)(hv >> 32); H[2] = pos < 64 ? (pos > 54 ? h10 >> (64 - pos) : 0u) : (h10 << (pos - 64));
    L[0] = (u32)lv; L[1] = (u32)(lv >> 32); L[2] = pos < 64 ? (pos > 54 ? l10 >> (64 - pos) : 0u) : (l10 << (pos - 64));
#pragma unroll
    for (int o = 1; o < 8; o <<= 1) {
#pragma unroll
        for (int k = 0; k < 3; ++k) {
            H[k] |= __shfl_xor_sync(0xFFFFFFFFu, H[k], o);
            L[k] |= __shfl_xor_sync(0xFFFFFFFFu, L[k], o);
        }
        bs += __shfl_xor_sync(0xFFFFFFFFu, bs, o);
    }
    bs_out = bs;
    flags_out = block_flags(H, L);
}

// The summaries of blocks 0 .. n-1 into info[2i] (sum |x-mid|) and info[2i+1] (flags), block i starting at blk(i): passes
// of 32 blocks, one lane per block. A last pass of at most four blocks runs eight lanes per block (block_scan_split8)
// when split_ok: those blocks lie one after another from a 4-byte aligned blk(i). vec_ok: every blk(i) is 16-byte aligned.
template <class Blk>
__device__ __forceinline__ void block_pass(Blk blk, u32 n, bool split_ok, bool vec_ok, u32 mid, u32 a_thl, u32 b_thl, u32 *info,
                                           int lane) {
    for (u32 i0 = 0; i0 < n; i0 += 32) {
        const u32 left = n - i0;
        u32 bs, fl;
        if (left <= 4u && split_ok) {
            block_scan_split8(blk(i0), lane, left, mid, a_thl, b_thl, bs, fl);
            const u32 i = i0 + (u32)(lane >> 3);
            if ((lane & 7) == 0 && (u32)(lane >> 3) < left) { info[2 * i] = bs; info[2 * i + 1] = fl; }
        } else if ((u32)lane < left) {
            const u32 i = i0 + (u32)lane;
            block_scan(blk(i), vec_ok, mid, a_thl, b_thl, bs, fl);
            info[2 * i] = bs; info[2 * i + 1] = fl;
        }
    }
}

// dst[0, len) = src[0, len) by one warp: 16-byte copies when both sides are 16-byte aligned
__device__ __forceinline__ void warp_copy(u16 *dst, const u16 *src, u32 len, int lane) {
    if (((reinterpret_cast<uintptr_t>(src) | reinterpret_cast<uintptr_t>(dst)) & 15) == 0) {
        const u32 nv = len >> 3;
        for (u32 i = lane; i < nv; i += 32) reinterpret_cast<uint4 *>(dst)[i] = reinterpret_cast<const uint4 *>(src)[i];
        for (u32 i = 8 * nv + lane; i < len; i += 32) dst[i] = src[i];
    } else {
        for (u32 i = lane; i < len; i += 32) dst[i] = src[i];
    }
}

// Start staging samples [first, first+count) of the batch into `buf` (bulk async copy when the batch base is 16-byte
// aligned, plain loads otherwise); completion is one phase of `bar` either way. Returns the sample index of `first`
// inside buf.
__device__ __forceinline__ int chunk_issue(unsigned char *buf, const u16 *pcm, size_t total_bytes, bool base_aligned,
                                           size_t first, u32 count, u64 *bar, int lane) {
    const size_t lo = first * 2, hi = lo + (size_t)count * 2;
    if (base_aligned) {
        const size_t lo_al = lo & ~(size_t)15;
        size_t hi_al = (hi + 15) & ~(size_t)15;
        const size_t lim = total_bytes & ~(size_t)15;
        if (hi_al > lim) hi_al = lim;
        const int shift = (int)((lo - lo_al) >> 1);
        if (hi > hi_al) {                                        // tail beyond the last whole 16-byte granule
            const u16 *g = reinterpret_cast<const u16 *>(reinterpret_cast<const unsigned char *>(pcm) + hi_al);
            u16 *d = reinterpret_cast<u16 *>(buf + (hi_al - lo_al));
            const int n = (int)((hi - hi_al) >> 1);
            if (lane < n) d[lane] = g[lane];
        }
        __syncwarp();
        if (lane == 0) {
            const u32 nbytes = (u32)(hi_al - lo_al);
            mbar_arrive_expect_tx(bar, nbytes);
            bulk_g2s(buf, reinterpret_cast<const unsigned char *>(pcm) + lo_al, nbytes, bar);
        }
        return shift;
    }
    const u16 *g = pcm + first;
    u16 *d = reinterpret_cast<u16 *>(buf);
    for (u32 i = lane; i < count; i += 32) d[i] = g[i];
    __syncwarp();
    if (lane == 0) mbar_arrive(bar);
    return 0;
}

// position of the first set bit at index >= from in a bitmap held one 32-bit word per lane; -1 if none
__device__ __forceinline__ int find_first(u32 word, int lane, int from) {
    const int fw = from >> 5, fb = from & 31;
    u32 m = lane > fw ? word : (lane == fw ? (word & (0xFFFFFFFFu << fb)) : 0u);
    if (from >= 1024) m = 0;
    const u32 bal = __ballot_sync(0xFFFFFFFFu, m != 0);
    if (!bal) return -1;
    const int L = __ffs(bal) - 1;
    const u32 mw = __shfl_sync(0xFFFFFFFFu, m, L);
    return 32 * L + __ffs(mw) - 1;
}
// bitmap shift towards index 0: result[i] = x[i+s], 0 < s < 32
__device__ __forceinline__ u32 bm_shr(u32 x, int s, int lane) {
    u32 nxt = __shfl_down_sync(0xFFFFFFFFu, x, 1);
    if (lane == 31) nxt = 0;
    return (x >> s) | (nxt << (32 - s));
}


// ---- frames from block summaries ---------------------------------------------------------------------------------
// One pass over up to 32 frames k0 + lane (frame k = blocks k, k+1; info[2*blk] = sum |x-mid|, info[2*blk+1] = flags of
// block_flags). `cin` is the class of the last out-of-band sample in the blocks before k0 (0 at the start of a capture)
// and is advanced to cover the blocks of the frames handled here (lanes with k >= kend contribute nothing), so passes
// may start at any frame and stop anywhere: the streaming kernels resume where the previous push ended.
// Frames are absolute (k == 0 is the capture's first frame); info holds the summaries of blocks koff, koff + 1, ... (0: all
// of them from block 0), so a caller may keep only the blocks of the frames at hand.
// Returns the ballot of "frame active" (VAD.C:164) over the 32 lanes.
__device__ __forceinline__ u32 frames_pass(const u32 *info, u32 k0, u32 kend, int lane, const atap_tag &at, u32 &cin, u32 koff) {
    const u32 k = k0 + (u32)lane;
    const bool ok = k < kend;
    u32 bs0 = 0, f0 = 0, bs1 = 0, f1 = 0;
    const u32 j = k - koff;
    if (ok) { bs0 = info[2 * j]; f0 = info[2 * j + 1]; bs1 = info[2 * j + 2]; f1 = info[2 * j + 3]; }
    const u32 zc0 = f0 & 127u, lc0 = (f0 >> 7) & 3u, lcA0 = (f0 >> 9) & 3u, p00 = (f0 >> 11) & 1u;
    const u32 zc1 = f1 & 127u, lc1 = (f1 >> 7) & 3u;
    const u32 fc0 = lc0 ? ((zc0 & 1u) ? 3u - lc0 : lc0) : 0u;      // first class from last class + parity
    const u32 fc1 = lc1 ? ((zc1 & 1u) ? 3u - lc1 : lc1) : 0u;
    // inclusive "last out-of-band class" scan over the blocks of this pass
    u32 inc = lc0;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const u32 up = __shfl_up_sync(0xFFFFFFFFu, inc, o);
        if (lane >= o && inc == 0) inc = up;
    }
    if (inc == 0) inc = cin;
    u32 prev = __shfl_up_sync(0xFFFFFFFFu, inc, 1);               // carry of block k-1
    if (lane == 0) prev = cin;
    cin = __shfl_sync(0xFFFFFFFFu, inc, 31);
    const u32 init = k == 0 ? 0u : (lcA0 ? lcA0 : prev);          // class of last out-of-band sample <= i+78
    u32 zc = zc0 + zc1 + ((lc0 && fc1 && lc0 != fc1) ? 1u : 0u);
    const u32 F = fc0 ? fc0 : fc1;
    const bool pos1 = fc0 ? (p00 == 0) : (fc1 != 0);              // first out-of-band sample not at position 0
    if (pos1 && init != 0 && init != F) ++zc;
    const bool active = ok && ((bs0 + bs1) > at.s_thl || zc > at.z_thl);   // VAD.C:164
    return __ballot_sync(0xFFFFFFFFu, active);
}

// ---- the endpoint FSM, carried across windows ------------------------------------------------------------------
// position of the last set bit in a bitmap held one 32-bit word per lane; -1 if none
__device__ __forceinline__ int find_last(u32 word) {
    const u32 bal = __ballot_sync(0xFFFFFFFFu, word != 0);
    if (!bal) return -1;
    const int L = 31 - __clz(bal);
    const u32 mw = __shfl_sync(0xFFFFFFFFu, word, L);
    return 32 * L + 31 - __clz(mw);
}

// The FSM's state between windows: open (a segment has opened and not closed), closed = the n segments before it, and
// run = the length of the run at the end of the frames seen so far that the FSM is counting (active frames while
// closed, inactive ones while open), always shorter than the 8 / 11 that would complete it.
struct LongFsm {
    bool open;
    u32 n, run;
};

// The endpoint FSM (VAD.C:164-216) over one window of nw <= 1024 frames starting at frame `base` (activity bitmap aw,
// one 32-frame word per lane), continuing from state f: 8 consecutive active frames open a segment at the first of them,
// 11 consecutive inactive frames close it at the first of those. A run carried in from the previous window completes at
// the window's first frames; later runs are found with bit tricks (a8 / z11 below, find_first). Windows may have any
// length up to 1 024: a run longer than the window is carried on, and frames past the window are unknown, so after any
// window f holds exactly the decisions the sequential FSM has taken by its last frame. Every lane calls
// act.open(lane, f.n, frame) when segment f.n opens at `frame` (VAD.C:178: start = 80 * frame) and act.close(lane, f.n,
// frame) when it closes with its first inactive frame at `frame` (VAD.C:201: end = 80 * frame + 80); f is updated after
// the call. There is no limit on the number of segments: an act that keeps SR_MAX_VC_CON ignores the later ones.
template <class Act>
__device__ __forceinline__ void long_fsm_window(u32 aw, u32 nw, u32 base, int lane, LongFsm &f, Act &act) {
    const u32 fullw = nw >> 5, rem = nw & 31u;
    const u32 vmask = (u32)lane < fullw ? 0xFFFFFFFFu : ((u32)lane == fullw ? ((1u << rem) - 1u) : 0u);
    aw &= vmask;
    const u32 z = ~aw & vmask;
    u32 a8 = aw & bm_shr(aw, 1, lane);
    a8 &= bm_shr(a8, 2, lane);
    a8 &= bm_shr(a8, 4, lane);                                     // a8[i]: frames i..i+7 all active
    u32 z8 = z & bm_shr(z, 1, lane);
    z8 &= bm_shr(z8, 2, lane);
    z8 &= bm_shr(z8, 4, lane);
    const u32 z11 = z8 & bm_shr(z8, 3, lane);                      // z11[i]: frames i..i+10 all inactive
    auto open_at = [&](u32 frame) {
        act.open(lane, f.n, frame);
        f.open = true;
    };
    auto close_at = [&](u32 frame) {
        act.close(lane, f.n, frame);
        ++f.n;
        f.open = false;
    };
    int cur = 0;                                                   // where the search for the next event resumes
    bool event = false;
    if (f.run) {                                                   // a run that began in the previous window
        const u32 need = (f.open ? 11u : 8u) - f.run, msk = (1u << need) - 1u;
        const u32 w0 = __shfl_sync(0xFFFFFFFFu, f.open ? z : aw, 0);
        if (need <= nw && (w0 & msk) == msk) {
            if (f.open) close_at(base - f.run); else open_at(base - f.run);
            cur = (int)need;                                       // the opening / closing frame + 8 / + 11
            event = true;
        }
    }
    for (;;) {
        const int p = find_first(f.open ? z11 : a8, lane, cur);
        if (p < 0) break;
        if (f.open) { close_at(base + (u32)p); cur = p + 11; } else { open_at(base + (u32)p); cur = p + 8; }
        event = true;
    }
    // the run at the end of the window: frames since the last one that breaks it (and since the last event)
    const int last_brk = find_last(f.open ? aw : z);
    if (!event && last_brk < 0) f.run += nw;
    else {
        const int from = max(last_brk + 1, cur);
        f.run = from < (int)nw ? nw - (u32)from : 0u;
    }
}

// ---- one window of frames: summaries -> activity -> FSM ----------------------------------------------------------
// Frames [k, k + nw), nw <= 1024, from the block summaries at info (block j at info[2 (j - koff)]): the activity words by
// frames_pass with last_sig carried in cin (VAD.C:121-164), then the endpoint FSM from state f (VAD.C:164-216).
template <class Act>
__device__ __forceinline__ void vad_window(const u32 *info, u32 koff, u32 k, u32 nw, int lane, const atap_tag &at, u32 &cin,
                                           LongFsm &f, Act &act) {
    u32 aw = 0;                                                    // lane j: activity of frames k + 32j .. + 31
    for (u32 j = 0; 32u * j < nw; ++j) {
        const u32 word = frames_pass(info, k + 32u * j, k + nw, lane, at, cin, koff);
        if ((u32)lane == j) aw = word;
    }
    long_fsm_window(aw, nw, k, lane, f, act);
}

// The FSM's actions for a capture of at most SR_MAX_VC_CON segments (K0, K4): lane j < 6 holds seg_off[j], the start of
// segment n in lane 2n and its end in lane 2n + 1. Later segments land in lanes that are never stored, or in none.
struct SegLanes {
    u32 seg;
    __device__ __forceinline__ void open(int lane, u32 n, u32 frame) {        // VAD.C:178
        if ((u32)lane == 2u * n) seg = 80u * frame;
    }
    __device__ __forceinline__ void close(int lane, u32 n, u32 frame) {       // VAD.C:201
        if ((u32)lane == 2u * n + 1u) seg = 80u * frame + 80u;
    }
};

// ---- what a streaming kernel carries and reports (K4 fixed captures, K14 live streams) ----------------------------
// The VAD state a stream carries from push to push: frames < `frames` are evaluated, cin is the class of the last
// out-of-band sample in blocks < frames (last_sig, VAD.C:99), f the endpoint FSM's state and open_start the start of the
// open segment (SR_SEG_NULL when none is open).
struct StreamVad {
    u32 frames, cin;
    LongFsm f;
    u32 open_start;
};

struct StreamEventDev {         // work list of the segments closed by the current push
    u32 stream, segment, start, end;
};

// A push's event list: one atomicAdd per closed segment, at most cap events kept
struct StreamEvents {
    StreamEventDev *ev;
    u32 *seg_ev, *map_ev, *n_ev;
    atap_tag *atap_ev;
    u32 cap;
    // segment n = [start, end) of stream s, which get_mfcc reads at offsets [ms, me) of PCM row s under at
    __device__ __forceinline__ void emit(u32 s, u32 n, u32 start, u32 end, u32 ms, u32 me, const atap_tag &at) const {
        const u32 e = atomicAdd(n_ev, 1u);
        if (e < cap) {
            StreamEventDev d; d.stream = s; d.segment = n; d.start = start; d.end = end;
            ev[e] = d;
            seg_ev[2 * e] = ms; seg_ev[2 * e + 1] = me;
            atap_ev[e] = at; map_ev[e] = s;
        }
    }
};

}  // namespace srk
