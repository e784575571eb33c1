// sr_vad_core.cuh -- warp-level building blocks of noise_atap (VAD.C:22-71) and VAD (VAD.C:97-218), shared by the
// batch kernel (sr_vad.cu: samples staged in shared memory) and the streaming kernel (sr_stream.cu: samples read from
// the streams' device rows): block summaries, the frame pass over summaries, and the endpoint FSM on the activity bitmap.
#pragma once
#include "sr_common.cuh"

namespace srk {

struct VadWarpView {
    const u16 *x;       // staged samples, x[0] = first sample of the utterance
    bool vec_ok;        // 16-byte aligned -> uint4 shared loads
};

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

// noise_atap's three sums (VAD.C:41-63) over staged samples x[0, n_len), n_len % 240 == 0: mid = sum/n_len,
// max_sum = sum over 240-sample blocks of max|x-mid|, abs_sum = sum |x-mid|. Vector form: lane l owns samples
// [80l, 80l+80) (three lanes per 240-block, n_len <= 2560), 16-byte loads, IDP.2A for the plain sum.
__device__ __forceinline__ void atap_stats(const u16 *x, bool vec_ok, u32 n_len, int lane, u32 &mid_out, u32 &max_sum_out,
                                           u32 &abs_sum_out) {
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
        const u32 mid = warp_sum(act ? s : 0u) / n_len;
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
        mid_out = mid;
        max_sum_out = warp_sum(bmax);
        abs_sum_out = warp_sum(sm);
        return;
    }
    u32 s = 0;
    for (u32 i = lane; i < n_len; i += 32) s += x[i];
    const u32 mid = warp_sum(s) / n_len;                             // VAD.C:41-45
    u32 max_sum = 0, abs_sum = 0;
    for (u32 i = 0; i < n_len; i += 240u) {                          // VAD.C:48-63
        u32 mx = 0, sm = 0;
        for (u32 h = lane; h < 240u; h += 32) { const u32 v = x[i + h], a = v > mid ? v - mid : mid - v; mx = max(mx, a); sm += a; }
        max_sum += warp_max(mx);
        abs_sum += sm;
    }
    mid_out = mid; max_sum_out = max_sum; abs_sum_out = warp_sum(abs_sum);
}

// the rest of noise_atap (VAD.C:65-70) from atap_stats' results: averages over the window, thresholds into at
__device__ __forceinline__ void atap_finish(atap_tag &at, u32 n_len, u32 mid, u32 max_sum, u32 abs_sum) {
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
__device__ __forceinline__ void block_scan(const VadWarpView &v, u32 i0, u32 mid, u32 a_thl, u32 b_thl, u32 &bs_out,
                                           u32 &flags_out) {
    u32 bs = 0;
    u32 H[3], L[3];
    const u16 *p = v.x + i0;
    if (mid <= 0xFFFFu) {
        u32 gA[3] = {0, 0, 0}, gB[3] = {0, 0, 0};      // "s >= a_thl", "s >= b_thl"; samples 0..31, 32..63, 64..79
        u32 bsx = 0, bsn = 0;
        const u32 mid2 = mid | (mid << 16), na = 0u - (a_thl << 16), nb = 0u - (b_thl << 16);
#pragma unroll
        for (int c = 0; c < 10; ++c) {
            u32 w[4];
            if (v.vec_ok) {
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
// may start at any frame and stop anywhere: the streaming kernel resumes where the previous push ended.
// Returns the ballot of "frame active" (VAD.C:164) over the 32 lanes.
__device__ __forceinline__ u32 frames_pass(const u32 *info, u32 k0, u32 kend, int lane, const atap_tag &at, u32 &cin) {
    const u32 k = k0 + (u32)lane;
    const bool ok = k < kend;
    u32 bs0 = 0, f0 = 0, bs1 = 0, f1 = 0;
    if (ok) { bs0 = info[2 * k]; f0 = info[2 * k + 1]; bs1 = info[2 * k + 2]; f1 = info[2 * k + 3]; }
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

// Endpoint FSM (VAD.C:164-216) on the activity bitmap of frames [0, nfr) held one 32-frame word per lane (nfr <= 1024):
// 8 consecutive active frames open a segment at the first of them, 11 consecutive inactive frames close it at the first
// of those; at most SR_MAX_VC_CON segments. Frames >= nfr are unknown (neither active nor inactive), so the result for a
// prefix of a capture is exactly the set of decisions the sequential FSM has taken after frame nfr-1.
__device__ __forceinline__ void fsm_segments(u32 aw, u32 nfr, int lane, u32 (&seg)[6]) {
    const u32 fullw = nfr >> 5, rem = nfr & 31u;
    const u32 vmask = (u32)lane < fullw ? 0xFFFFFFFFu : ((u32)lane == fullw ? ((1u << rem) - 1u) : 0u);
    aw &= vmask;
    u32 a8 = aw & bm_shr(aw, 1, lane);
    a8 &= bm_shr(a8, 2, lane);
    a8 &= bm_shr(a8, 4, lane);                                     // a8[i]: frames i..i+7 all active
    u32 z = ~aw & vmask;
    u32 z8 = z & bm_shr(z, 1, lane);
    z8 &= bm_shr(z8, 2, lane);
    z8 &= bm_shr(z8, 4, lane);
    const u32 z11 = z8 & bm_shr(z8, 3, lane);                      // z11[i]: frames i..i+10 all inactive
    int cur = 0;
    for (int sgi = 0; sgi < (int)SR_MAX_VC_CON; ++sgi) {
        const int pfr = find_first(a8, lane, cur);
        if (pfr < 0) break;
        seg[2 * sgi] = 80u * (u32)pfr;                             // VAD.C:178: i - 7*80 with i = 80*(pfr+7)
        const int q = find_first(z11, lane, pfr + 8);
        if (q < 0) break;                                          // never closes: end stays NULL
        seg[2 * sgi + 1] = 80u * (u32)q + 80u;                     // VAD.C:201: i - 11*80 + 160 with i = 80*(q+10)
        cur = q + 11;
    }
}

}  // namespace srk
