// sr_mfcc.cu -- K1: batched get_mfcc (Src/Speech_Recog/MFCC.C:86-191) with the bit-exact
// fixed-point radix-4 FFT of Src/BSP/cr4_fft_1024_stm32.s:95-281 done in registers/shared memory.
//
// Work decomposition (H100: 132 SMs, one persistent CTA per SM):
//   * a CTA walks utterances b = blockIdx.x, +gridDim.x, ...; each utterance's PCM segment
//     [start-1, end) is staged into a 3-deep shared-memory ring with 1-D bulk async copies (TMA
//     engine, cp.async.bulk + mbarrier complete_tx), one utterance ahead, as a side job that
//     rotates over the warps -- every PCM sample is read from HBM exactly once although frames
//     overlap by 50 %;
//   * all 16 warps take frames round-robin from the CTA's concatenated frame stream,
//     one frame per warp: pre-emphasis + Hamming (MFCC.C:115-124), FFT, |.| (MFCC.C:49-60),
//     energy (MFCC.C:128-133), 24 triangular filters (MFCC.C:136-162), log (MFCC.C:165-170),
//     DCT (MFCC.C:173-183) -> 12 x s16.
//
// FFT blocking (validated against the asm restatement by tools/fft_block_model.py):
//   stage 0 collapses for a real frame of <= 256 samples: y0[4*idx+m] = (w[bitrev8(idx)]>>2, 0);
//   block A (G,q1): 4 stage-1 butterflies (groups 4G+m2) + 4 stage-2 butterflies (q2=q1+4*m1)
//                   on 16 register-resident points, 64 blocks/frame = 2 per lane;
//   exchange through a padded shared buffer, one 64-bit (re, im) word pair per point (conflict-free both ways:
//                   a 64-bit access is two half-warp wavefronts, and in each half-warp point slot padF(e) mod 16 is
//                   4G + q1 for the stores and 16 consecutive values for the loads);
//   block B (q3):   4 stage-3 butterflies (groups m4) + 4 stage-4 butterflies (q4=q3+64*m3),
//                   only output legs 0,1 (bins < 512, MFCC.C:49) are formed.
//
// s16 stores without wrap: the asm stores every stage result with STRH (low 16 bits). On THIS path the
// wrap can never trigger: the stage-0 outputs are real with |.| <= 8192 (an s16 sample >> 2); a radix-4
// stage maps complex magnitudes <= M to magnitudes <= (M + 3*1.00015*M)/4 + 3 (twiddle rounding
// |W| <= 1.00015, a few LSB of floor rounding), so after four stages every component is <= 8209 << 32767
// and the sign-extending truncation is the identity (also no 32-bit overflow: 2*8209*16385 < 2^31).
// The generic kernel below runs the shared core's FFT, which keeps the wrap because it accepts arbitrary complex input.
#include <stdio.h>
#include "sr_mfcc_core.cuh"

namespace srk {

constexpr int kPcmBufBytes = 19264;          // (118*80+160+1)*2 = 19202 B + 16 B alignment slack, /64
__host__ __device__ constexpr int padF(int e) { return e + ((e >> 6) << 2); }
// FFT data: 1024 points + 4 pad points per 64, two words each; the filter-stage scratch (sr_common.cuh) overlays it
constexpr int kFftWords = 2 * (padF(1023) + 1);   // 2168
static_assert(kFftWords >= kFftWordsTotal, "filter scratch must fit in the FFT buffer");

constexpr int kMfccWarps = 16;               // every warp takes frames and stages utterances as a side job
constexpr int kNBuf = 3;                     // PCM ring depth

struct __align__(16) MfccSmem {
    unsigned char pcm[kNBuf][kPcmBufBytes];
    int2 tw[340 * 3];
    u32 log_thr[2220];
    u32 tri_even[512];                       // filter weights as 32-bit words: no unpacking in the frame loop
    u32 tri_odd[512];
    int4 dct[24 * 3];                        // DCT role of lane l < 24: its 12 weights as three 16-byte rows (12-word stride: conflict-free)
    u32 fftbuf[kMfccWarps][kFftWords];
    s32 wq[kMfccWarps][160];
    u32 lg[kMfccWarps][32];
    u64 full[kNBuf];
    u64 empty[kNBuf];
    s32 meta[kNBuf][5];                      // {F (-1 = no more utterances), sample index of x[start-1] in the buffer, mid, utterance b,
                                             //  x[start-1] pinned to mid (start == 0)}
    int turn;                                // dynamic hand-out: number of the CTA's next claim (claims are made in ring order)
};

static_assert(sizeof(MfccSmem) <= 232448, "mfcc_kernel_s16 exceeds the 227 KB shared-memory opt-in limit");

// Stage utterance number `it` of this CTA's walk (batch row b) into ring slot it % kNBuf: one warp, lane 0 issues
// the bulk copy. Bytes [lo,hi) of the batch = samples start-1 .. start+80(F-1)+159 of the utterance.
// x[-1] of a segment that starts at sample 0 (MFCC.C:119, i = 0) is not a sample of the utterance: it is the last
// sample of the previous row, or lies before the batch. Every batched entry point pins it to the utterance's own mid
// (its pre-emphasis term is then 0), so an utterance's features do not depend on its row, its chunk, its shard or
// another stream. The slot only flags it (meta[s][4]); the warp that takes frame 0 writes mid over x[0] once the slot
// is full. A store here could be overwritten by the bulk copy, which spans x[-1] when sample 0 is not 16-byte aligned.
__device__ __forceinline__ void stage_utterance(MfccSmem &sm, int it, u32 b, const u16 *__restrict__ pcm,
                                                u32 U, const u32 *__restrict__ seg, u32 seg_stride,
                                                const atap_tag *__restrict__ atap, unsigned char *__restrict__ ftr,
                                                const u32 *__restrict__ row_map, size_t total_bytes, bool base_aligned,
                                                int lane) {
    const int s = it % kNBuf;
    const u32 st = seg[(size_t)b * seg_stride], en = seg[(size_t)b * seg_stride + 1];
    const u32 mid = atap[b].mid_val;
    const long long row = row_map ? (long long)row_map[b] : (long long)b;
    if (it >= kNBuf) mbar_wait(&sm.empty[s], ((it / kNBuf) - 1) & 1);
    const int F = mfcc_frames<SR_FRAME_LEN>(st, en, U);
    if (lane == 0) *reinterpret_cast<u16 *>(ftr + (size_t)b * kFtrBytes + 2) = (u16)F;   // MFCC.C:106,189
    if (F == 0) {
        if (lane == 0) {
            sm.meta[s][0] = 0; sm.meta[s][1] = 0; sm.meta[s][2] = (s32)mid; sm.meta[s][3] = (s32)b; sm.meta[s][4] = 0;
            mbar_arrive(&sm.full[s]);
        }
        return;
    }
    if (lane == 0) sm.meta[s][4] = (st == 0);
    long long first = row * U + st - 1;                    // -1 for row 0, start 0
    const long long last = row * U + st + 80ll * (F - 1) + 160;   // exclusive
    unsigned char *dst = sm.pcm[s];
    int off = 0;
    if (first < 0) {                                       // x[-1] would lie before the batch: copy from sample 0, which
        first = 0; off = 8;                                // lands at dst+16 (index 8); x[-1] is index 7, written by a consumer
        dst += 16;
    }
    const size_t lo = (size_t)first * 2, hi = (size_t)last * 2;
    if (base_aligned) {
        const size_t lo_al = lo & ~(size_t)15;
        size_t hi_al = (hi + 15) & ~(size_t)15;
        const size_t lim = total_bytes & ~(size_t)15;
        if (hi_al > lim) hi_al = lim;
        const u32 nbytes = (u32)(hi_al - lo_al);
        const int shift = (int)((lo - lo_al) >> 1);
        if (lane == 0) {
            sm.meta[s][0] = F; sm.meta[s][2] = (s32)mid; sm.meta[s][3] = (s32)b;
            sm.meta[s][1] = (off ? 7 : shift);             // index of x[start-1] (7 = slot just below dst+16)
        }
        // tail beyond the last whole 16-byte granule of the allocation: plain loads
        if (hi > hi_al) {
            const u16 *g = reinterpret_cast<const u16 *>(reinterpret_cast<const unsigned char *>(pcm) + hi_al);
            u16 *d = reinterpret_cast<u16 *>(dst + (hi_al - lo_al));
            const int n = (int)((hi - hi_al) >> 1);
            if (lane < n) d[lane] = g[lane];
        }
        __syncwarp();
        if (lane == 0) {
            mbar_arrive_expect_tx(&sm.full[s], nbytes);
            bulk_g2s(dst, reinterpret_cast<const unsigned char *>(pcm) + lo_al, nbytes, &sm.full[s]);
        }
    } else {                                               // unaligned batch base: cooperative plain copy
        const u16 *g = pcm + first;
        u16 *d = reinterpret_cast<u16 *>(dst);
        const int n = (int)(last - first);
        for (int i = lane; i < n; i += 32) d[i] = g[i];
        __syncwarp();
        if (lane == 0) {
            sm.meta[s][0] = F; sm.meta[s][2] = (s32)mid; sm.meta[s][1] = off ? 7 : 0; sm.meta[s][3] = (s32)b;
            mbar_arrive(&sm.full[s]);
        }
    }
}

// end-of-work marker in ring slot it % kNBuf: consumers leave their loop when they meet it
__device__ __forceinline__ void stage_end(MfccSmem &sm, int it, int lane) {
    const int s = it % kNBuf;
    if (it >= kNBuf) mbar_wait(&sm.empty[s], ((it / kNBuf) - 1) & 1);
    if (lane == 0) { sm.meta[s][0] = -1; mbar_arrive(&sm.full[s]); }
}

// One persistent CTA per SM (threads per CTA are capped at floor(65536 / regs / 128) * 128). Every warp is a consumer,
// and the staging of utterance it+kAhead is a side job of warp it % kMfccWarps at the top of iteration it, so all four
// schedulers of the SM carry the same number of working warps.
// Measured and dropped: the asm's 3-multiply twiddle form (one IMAD traded for a subtract: 4.91 ms vs 4.76), forcing the
// C+-D sums of the butterflies onto the ALU pipe as three-input adds (4.86 vs 4.76), two 16-bit
// stores instead of PRMT + one 32-bit store in block A (4.86 vs 4.80), 20 warps @ 96 regs (5.29 ms vs 5.31), 24 warps @ 80 regs (5.48 ms) -- the half-rate ALU and
// FMA-heavy pipes, not occupancy, bound the kernel. On the H100 (400 W), no gain beyond run-to-run spread: storing w>>4 for
// stage 1's A leg to skip its shift (4 SASS instructions per frame fewer), and log100 as one correction step each way
// instead of the two loops (MFCC kernel 5.18 and 5.18 ms vs 5.20). Slower: 15 consumer warps plus a dedicated producer
// warp, which leaves one scheduler with 3 working warps (5 % on the B200; on the H100 (700 W) MFCC kernel 4.97 ms vs 4.74,
// step 6.01 ms vs 5.78).
__global__ void __maxnreg__(128) mfcc_kernel_s16(const u16 *__restrict__ pcm, u32 U, u32 B, const u32 *__restrict__ seg,
                                                 u32 seg_stride, const atap_tag *__restrict__ atap,
                                                 unsigned char *__restrict__ ftr, const DevTables *__restrict__ tab,
                                                 const u32 *__restrict__ row_map, u32 rows_total, const u32 *__restrict__ B_dev,
                                                 u32 *__restrict__ work /* [0] next utterance to hand out, [1] CTAs finished; NULL: static */) {
    constexpr int kAhead = kNBuf - 2;                      // slot of it+kAhead was last used by utterance it-2
    if (B_dev) B = min(B, *B_dev);                         // batch size produced on the device (streaming: segments closed by this push)
    // the last CTA out re-arms the hand-out counters for the next launch on this stream
    auto cta_done = [&]() {
        if (work && threadIdx.x == 0) {
            __threadfence();
            if (atomicAdd(&work[1], 1u) == gridDim.x - 1u) { work[0] = 0; work[1] = 0; }
        }
    };
    if (blockIdx.x >= B) { cta_done(); return; }           // more CTAs than utterances (device-side batch size): these never claim
    extern __shared__ __align__(128) unsigned char smem_raw[];
    MfccSmem &sm = *reinterpret_cast<MfccSmem *>(smem_raw);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

    // ---- one-time: tables to shared memory, barriers ------------------------------------------
    for (int i = threadIdx.x; i < 340 * 3; i += blockDim.x) sm.tw[i] = tab->tw[i];
    for (int i = threadIdx.x; i < 2220; i += blockDim.x) sm.log_thr[i] = tab->log_thr[i];
    // filter weights in the same bank-swizzled row layout as the running totals (flt_word): a lane reads its 16 weights with
    // four 16-byte loads, and eight neighbouring lanes hit 32 distinct banks (plain 16-word rows would conflict 4-way)
    for (int i = threadIdx.x; i < 24 * 12; i += blockDim.x)
        reinterpret_cast<s32 *>(sm.dct)[i] = (s32)tab->dct[(i / 24) * 24 + ((i / 12) & 1) * 12 + i % 12];
    for (int i = threadIdx.x; i < 512; i += blockDim.x) {
        sm.tri_even[flt_word(i >> 4, i & 15)] = tab->tri_even[i];
        sm.tri_odd[flt_word(i >> 4, i & 15)] = tab->tri_odd[i];
    }
    if (threadIdx.x == 0) {
        for (int s = 0; s < kNBuf; ++s) { mbar_init(&sm.full[s], 1); mbar_init(&sm.empty[s], kMfccWarps); }
        sm.turn = 0;
        mbar_fence_init();
    }
    __syncthreads();

    // row_map (streaming): utterance b's samples live in PCM row row_map[b] of a [rows_total][U] buffer
    const size_t total_bytes = (size_t)(row_map ? rows_total : B) * U * 2;
    const bool base_aligned = (reinterpret_cast<uintptr_t>(pcm) & 15) == 0;

    // Utterances are handed out dynamically (one atomic per utterance per CTA) when `work` is given: CTAs whose utterances
    // happen to hold more frames, or that start late, take fewer; statically strided CTAs ended up to 2 % apart.
    // Stage utterance number `it_s` of this CTA's sequence (or the end marker), executed by one warp.
    // The claims of one CTA are made by different warps, so they take turns in ring order: the counter only grows, hence
    // the utterance numbers of a CTA grow with it_s and every slot behind an end marker holds an end marker too (a later
    // slot claimed EARLIER could hold a real utterance that the consumers, leaving at the first marker, would never see).
    // A claim waits only for the claim before it, which is made at the top of an earlier iteration: no cycle.
    auto claim_stage = [&](int it_s) {
        u32 b;
        if (work) {
            b = 0;
            if (lane == 0) {
                volatile int *turn = &sm.turn;
                while (*turn != it_s) { }
                b = atomicAdd(&work[0], 1u);
                __threadfence_block();
                if (b != 0xFFFFFFFFu) *turn = it_s + 1;                    // (the test makes the store wait for the atomic's result)
            }
            b = __shfl_sync(0xFFFFFFFFu, b, 0);
        }
        else b = blockIdx.x + (u32)it_s * gridDim.x;
        if (b < B) stage_utterance(sm, it_s, b, pcm, U, seg, seg_stride, atap, ftr, row_map, total_bytes, base_aligned, lane);
        else stage_end(sm, it_s, lane);
    };
    if (warp < kAhead) claim_stage(warp);                 // prologue: utterances 0 .. kAhead-1

    u32 *fb = sm.fftbuf[warp];
    s32 *wq = sm.wq[warp];
    const int q1 = lane & 3;
    // stage-1 twiddles (table block N=16, triple q1: legs K2 -> p2, K1 -> p1; leg 3 is all-zero)
    const int2 k1_2 = sm.tw[q1 * 3 + 1], k1_1 = sm.tw[q1 * 3 + 2];
    // stage-2 twiddles (block N=64, triple q2 = q1 + 4*m1): the same for both passes and every frame
    int2 k2t[4][3];
#pragma unroll
    for (int m1 = 0; m1 < 4; ++m1)
#pragma unroll
        for (int j = 0; j < 3; ++j) k2t[m1][j] = sm.tw[(4 + q1 + 4 * m1) * 3 + j];
    const u32 hm0 = tab->hamm[lane], hm1 = tab->hamm[lane + 32], hm2 = tab->hamm[lane + 64],
              hm3 = tab->hamm[lane + 96], hm4 = tab->hamm[lane + 128];
    // filter role: lanes 0..23 -> filter h = lane: S(hi) - S(lo) of its parity's prefix sums (see DevTables)
    const int fsw = (lane >> 1) & 3;                       // bank swizzle of the running-total rows (flt_word)
    int fe_lo = kFltZero, fe_hi = kFltZero, fx_lo = kFltX, fx_hi = kFltX;
    if (lane < 24) {
        fe_lo = tab->flt_e_lo[lane]; fe_hi = tab->flt_e_hi[lane];
        fx_lo = kFltX + (lane & 1) * 33 + tab->flt_x_lo[lane]; fx_hi = kFltX + (lane & 1) * 33 + tab->flt_x_hi[lane];
    }
    // DCT role: lanes 0..23 -> coefficient c = lane>>1, half = lane&1 (12 filters each); lanes 24..31 compute a discarded copy
    const int4 *dctk4 = sm.dct + 3 * (lane < 24 ? lane : 0);

    u32 gidx = 0;   // frames of this CTA's stream before the current utterance
    for (int it = 0;; ++it) {
        if (warp == it % kMfccWarps) claim_stage(it + kAhead);
        const int s = it % kNBuf;
        mbar_wait(&sm.full[s], (it / kNBuf) & 1);
        const int F = sm.meta[s][0];
        if (F < 0) break;                                                  // end marker: no more utterances for this CTA
        const u32 b = (u32)sm.meta[s][3];
        const int off = sm.meta[s][1];
        const s32 mid = sm.meta[s][2];
        u16 *x = reinterpret_cast<u16 *>(sm.pcm[s]) + off;               // x[0] = sample start-1
        unsigned char *out_rows = ftr + (size_t)b * kFtrBytes + 4;
        const int f0 = (int)((warp - (int)(gidx % kMfccWarps) + kMfccWarps) % kMfccWarps);   // this warp's first frame
        // start == 0: x[-1] := mid (see stage_utterance). Only frame 0 reads x[0], and only its lane 0.
        if (f0 == 0 && lane == 0 && sm.meta[s][4]) x[0] = (u16)mid;

        // pre-emphasis + Hamming, MFCC.C:115-124, of the frame at xf (xf[i] = vc_dat[i-1]); keeps w>>2 (stage-0 output) in wq
        auto preemph = [&](const u16 *xf) {
            const u32 hm[5] = {hm0, hm1, hm2, hm3, hm4};
#pragma unroll
            for (int k = 0; k < 5; ++k) {
                const int i = lane + 32 * k;
                wq[i] = preemph_hamm(xf[i + 1], xf[i], (u32)mid, hm[k]) >> 2;   // BUTFLY4ZERO_OPT with B=C=D=0
            }
        };
        for (int f = f0; f < F; f += kMfccWarps) {
            const u16 *xf = x + 80 * f;                                  // xf[i] = vc_dat[i-1]
            preemph(xf);
            __syncwarp();

            // ---- block A: stages 1+2 -----------------------------------------------------------
#pragma unroll 1
            for (int pass = 0; pass < 2; ++pass) {
                const int G = (lane >> 2) + 8 * pass;
                const int r0 = (int)(__brev((u32)G) >> 28);
                u32 vr[4][4], vi[4][4];                                    // [m2][m1]
#pragma unroll
                for (int m2 = 0; m2 < 4; ++m2) {
                    const int r = r0 + 16 * (((m2 & 1) << 1) | (m2 >> 1));
                    const u32 a = (u32)wq[r];
                    const u32 c = (u32)wq[r + 64];
                    u32 Cr, Ci, Br = 0, Bi = 0;
                    cxmul(Cr, Ci, c, 0u, (u32)k1_2.x, (u32)k1_2.y);
                    if ((m2 & 1) == 0) {                                   // r+128 < 160 only for r < 32
                        const u32 bb = (u32)wq[r + 128];
                        cxmul(Br, Bi, bb, 0u, (u32)k1_1.x, (u32)k1_1.y);
                    }
                    u32 o[8];
                    cxadda4<14>(a, 0u, Br, Bi, Cr, Ci, 0u, 0u, o[0], o[1], o[2], o[3], o[4], o[5], o[6], o[7]);
#pragma unroll
                    for (int m1 = 0; m1 < 4; ++m1) { vr[m2][m1] = o[2 * m1]; vi[m2][m1] = o[2 * m1 + 1]; }   // STRH wrap is the identity here (|.| <= 8209, see header)
                }
#pragma unroll
                for (int m1 = 0; m1 < 4; ++m1) {
                    const int q2 = q1 + 4 * m1;
                    const int2 k3 = k2t[m1][0], k2 = k2t[m1][1], k1 = k2t[m1][2];
                    u32 Dr, Di, Cr, Ci, Br, Bi;
                    cxmul(Dr, Di, vr[3][m1], vi[3][m1], (u32)k3.x, (u32)k3.y);
                    cxmul(Cr, Ci, vr[2][m1], vi[2][m1], (u32)k2.x, (u32)k2.y);
                    cxmul(Br, Bi, vr[1][m1], vi[1][m1], (u32)k1.x, (u32)k1.y);
                    u32 o[8];
                    cxadda4<14>(vr[0][m1], vi[0][m1], Br, Bi, Cr, Ci, Dr, Di, o[0], o[1], o[2], o[3], o[4], o[5], o[6], o[7]);
                    // point e = 64G + q2 + 16m as two words (re, im) at point slot padF(e): one 64-bit store, no packing
                    uint2 *dst = reinterpret_cast<uint2 *>(fb) + padF(64 * G + q2);
#pragma unroll
                    for (int m = 0; m < 4; ++m) dst[16 * m] = make_uint2(o[2 * m], o[2 * m + 1]);
                }
            }
            __syncwarp();

            // ---- block B: stages 3+4, magnitude, energy ---------------------------------------
            // Energy of bin k goes to word padF(k) (the filter stage's layout), which overlays points other lanes read:
            // each pass stores its energies only after every lane has read its points, pass 0's are held until then.
            u32 held[8];
#pragma unroll
            for (int pass = 0; pass < 2; ++pass) {
                const int q3 = lane + 32 * pass;
                u32 vr[4][4], vi[4][4];                                    // [m4][m3]
                const int2 *k = &sm.tw[(20 + q3) * 3];
                const int2 k3 = k[0], k2 = k[1], k1 = k[2];
                const uint2 *pts = reinterpret_cast<const uint2 *>(fb) + padF(q3);   // padF(256m4 + 64m3 + q3) = padF(q3) + padF(256m4 + 64m3)
#pragma unroll
                for (int m4 = 0; m4 < 4; ++m4) {
                    u32 pr[4], pi[4];
#pragma unroll
                    for (int m3 = 0; m3 < 4; ++m3) {
                        const uint2 p = pts[padF(256 * m4 + 64 * m3)];
                        pr[m3] = p.x; pi[m3] = p.y;
                    }
                    u32 Dr, Di, Cr, Ci, Br, Bi;
                    cxmul(Dr, Di, pr[3], pi[3], (u32)k3.x, (u32)k3.y);
                    cxmul(Cr, Ci, pr[2], pi[2], (u32)k2.x, (u32)k2.y);
                    cxmul(Br, Bi, pr[1], pi[1], (u32)k1.x, (u32)k1.y);
                    u32 o[8];
                    cxadda4<14>(pr[0], pi[0], Br, Bi, Cr, Ci, Dr, Di, o[0], o[1], o[2], o[3], o[4], o[5], o[6], o[7]);
#pragma unroll
                    for (int m3 = 0; m3 < 4; ++m3) { vr[m4][m3] = o[2 * m3]; vi[m4][m3] = o[2 * m3 + 1]; }
                }
                __syncwarp();                                               // every lane has read this pass's points
                if (pass == 1) {
#pragma unroll
                    for (int m3 = 0; m3 < 4; ++m3) { fb[padF(lane + 64 * m3)] = held[2 * m3]; fb[padF(lane + 64 * m3 + 256)] = held[2 * m3 + 1]; }
                }
#pragma unroll
                for (int m3 = 0; m3 < 4; ++m3) {
                    const int q4 = q3 + 64 * m3;
                    const int2 *kk = &sm.tw[(84 + q4) * 3];
                    const int2 j3 = kk[0], j2 = kk[1], j1 = kk[2];
                    u32 Dr, Di, Cr, Ci, Br, Bi;
                    cxmul(Dr, Di, vr[3][m3], vi[3][m3], (u32)j3.x, (u32)j3.y);
                    cxmul(Cr, Ci, vr[2][m3], vi[2][m3], (u32)j2.x, (u32)j2.y);
                    cxmul(Br, Bi, vr[1][m3], vi[1][m3], (u32)j1.x, (u32)j1.y);
                    u32 o[8];
                    cxadda4<14>(vr[0][m3], vi[0][m3], Br, Bi, Cr, Ci, Dr, Di, o[0], o[1], o[2], o[3], o[4], o[5], o[6], o[7]);
                    // bins q4 (leg 0) and q4+256 (leg 1); legs 2,3 are bins >= 512, unused (MFCC.C:49)
                    const u32 m0 = mag10_small(o[0], o[1]);
                    const u32 m1 = mag10_small(o[2], o[3]);
                    if (pass == 0) { held[2 * m3] = m0 * m0; held[2 * m3 + 1] = m1 * m1; }   // MFCC.C:131 (u32 wrap)
                    else { fb[padF(q4)] = m0 * m0; fb[padF(q4 + 256)] = m1 * m1; }
                }
            }
            __syncwarp();

            // ---- triangular filters, MFCC.C:136-162: lane owns bins [16*lane, 16*lane+16) ------
            // acc[h] = sum over the filter's bins of (E[k]*tri[k])/100, u32 wrap. Per parity the per-bin terms become
            // prefix sums: a lane keeps the running totals of its 16 bins (written to the warp's scratch) and its total;
            // a filter is a difference of two prefix values (running totals + the lane totals in between) -- exact mod 2^32.
            {
                u32 E[16];
                const uint4 *e4 = reinterpret_cast<const uint4 *>(fb + 16 * lane + 4 * (lane >> 2));   // padF(16*lane)
#pragma unroll
                for (int j = 0; j < 4; ++j) { const uint4 v = e4[j]; E[4 * j] = v.x; E[4 * j + 1] = v.y; E[4 * j + 2] = v.z; E[4 * j + 3] = v.w; }
                __syncwarp();                                               // every lane holds its energies: fb is scratch now
                const uint4 *we4 = reinterpret_cast<const uint4 *>(sm.tri_even + 16 * lane);
                const uint4 *wo4 = reinterpret_cast<const uint4 *>(sm.tri_odd + 16 * lane);
                uint4 *re4 = reinterpret_cast<uint4 *>(fb + 16 * lane);                    // this lane's row, group g at slot g ^ fsw
                uint4 *ro4 = reinterpret_cast<uint4 *>(fb + kFltRowWords + 16 * lane);
                u32 te = 0, to = 0;
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    const uint4 we = we4[j ^ fsw], wo = wo4[j ^ fsw];
                    uint4 pe, po;                                           // running totals BEFORE bin 4j+c
                    pe.x = te; te += (E[4 * j] * we.x) / 100u;      po.x = to; to += (E[4 * j] * wo.x) / 100u;
                    pe.y = te; te += (E[4 * j + 1] * we.y) / 100u;  po.y = to; to += (E[4 * j + 1] * wo.y) / 100u;
                    pe.z = te; te += (E[4 * j + 2] * we.z) / 100u;  po.z = to; to += (E[4 * j + 2] * wo.z) / 100u;
                    pe.w = te; te += (E[4 * j + 3] * we.w) / 100u;  po.w = to; to += (E[4 * j + 3] * wo.w) / 100u;
                    re4[j ^ fsw] = pe; ro4[j ^ fsw] = po;
                }
                // lane totals as they are: the reader adds the few it spans (a 5-step warp scan of them -- ten dependent
                // shuffles per frame with four warps per scheduler -- measured 5 % slower)
                fb[kFltX + lane] = te;
                fb[kFltX + 33 + lane] = to;
                fb[kFltZero] = 0u;                                          // S(512)'s in-lane part (block A overwrote it)
            }
            __syncwarp();
            // ---- filter totals + log, MFCC.C:165-170 -------------------------------------------
            {
                // S(hi) - S(lo) = e_hi - e_lo + the totals of lanes [lo>>4, hi>>4): at most 6 of them (widest filter 85 bins),
                // independent predicated loads
                u32 acc = fb[fe_hi] - fb[fe_lo];
#pragma unroll
                for (int j = 0; j < 6; ++j) if (fx_lo + j < fx_hi) acc += fb[fx_lo + j];
                sm.lg[warp][lane] = (lane < 24) ? log100(acc, sm.log_thr) : 0u;
            }
            __syncwarp();
            // ---- DCT, MFCC.C:173-183 ---------------------------------------------------------
            {
                const int4 d0 = dctk4[0], d1 = dctk4[1], d2 = dctk4[2];
                const s32 dctk[12] = {d0.x, d0.y, d0.z, d0.w, d1.x, d1.y, d1.z, d1.w, d2.x, d2.y, d2.z, d2.w};
                dct_row(sm.lg[warp], dctk, out_rows + (size_t)f * kRowBytes, lane);
            }
            __syncwarp();
        }
        gidx += (u32)F;
        __syncwarp();
        if (lane == 0) mbar_arrive(&sm.empty[s]);
    }
    __syncthreads();                                   // every warp has made its last claim: only now may the counters be re-armed
    cta_done();
}

// ---- generic (unpruned) FFT + magnitude: the reference's global `fft` (MFCC.C:27-62) -----------
// One warp per frame, all five passes in shared memory exactly as the asm orders them. Not on the
// hot path; it exists for the secondary drop-in symbol and as an on-device cross-check of the
// pruned blocking above with arbitrary (complex, full-length) inputs.
__global__ void __launch_bounds__(128)
fft_generic_kernel(const u32 *__restrict__ in /*[n][1024] packed or NULL*/, const s16 *__restrict__ frames, u32 len,
                   u32 n, u32 *__restrict__ raw_out /*[n][1024] or NULL*/, u32 *__restrict__ mag /*[n][512] or NULL*/,
                   const DevTables *__restrict__ tab) {
    __shared__ u32 buf[4][1024];
    __shared__ u32 src[4][1024];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const u32 fr = blockIdx.x * 4 + warp;
    if (fr >= n) return;
    u32 *x = src[warp], *y = buf[warp];
    for (int i = lane; i < 1024; i += 32) {
        u32 v;
        if (in) v = in[(size_t)fr * 1024 + i];
        else v = (u32)i < len ? (u32)(u16)frames[(size_t)fr * len + i] : 0u;     // MFCC.C:37-45
        x[i] = v;
    }
    __syncwarp();
    fft_radix4<1024>(x, y, tab, lane);
    if (raw_out) for (int i = lane; i < 1024; i += 32) raw_out[(size_t)fr * 1024 + i] = y[i];
    if (mag) for (int i = lane; i < 512; i += 32) mag[(size_t)fr * 512 + i] = mag10(lo16s(y[i]), hi16s(y[i]));
}

// ---- host launchers -----------------------------------------------------------------------------
cudaError_t launch_mfcc(const u16 *pcm, u32 U, u32 B, const u32 *seg, u32 seg_stride, const atap_tag *atap,
                        void *ftr, int num_sms, cudaStream_t st, const u32 *row_map, u32 rows_total, const u32 *B_dev, u32 *work) {
    if (B == 0) return cudaSuccess;
    const DevTables *tab = dev_tables();
    if (!tab) return cudaErrorInitializationError;
    const size_t smem = sizeof(MfccSmem);
    const int threads = kMfccWarps * 32;
    cudaError_t e = cudaFuncSetAttribute(mfcc_kernel_s16, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
    const u32 grid = B < (u32)num_sms ? B : (u32)num_sms;
    mfcc_kernel_s16<<<grid, threads, smem, st>>>(pcm, U, B, seg, seg_stride, atap, static_cast<unsigned char *>(ftr), tab,
                                                 row_map, rows_total, B_dev, work);
    e = cudaGetLastError();
    if (e != cudaSuccess) {
        cudaFuncAttributes fa;
        if (cudaFuncGetAttributes(&fa, mfcc_kernel_s16) == cudaSuccess)
            fprintf(stderr, "mfcc kernel launch failed (%s): regs %d, maxThreads %d, static smem %zu, dyn smem %zu (max %d), threads %d\n",
                    cudaGetErrorString(e), fa.numRegs, fa.maxThreadsPerBlock, fa.sharedSizeBytes, smem,
                    fa.maxDynamicSharedSizeBytes, threads);
    }
    return e;
}

cudaError_t launch_fft_generic(const u32 *in_packed, const s16 *frames, u32 len, u32 n, u32 *raw_out, u32 *mag,
                               cudaStream_t st) {
    if (n == 0) return cudaSuccess;
    const DevTables *tab = dev_tables();
    if (!tab) return cudaErrorInitializationError;
    fft_generic_kernel<<<(n + 3) / 4, 128, 0, st>>>(in_packed, frames, len, n, raw_out, mag, tab);
    return cudaGetLastError();
}

}  // namespace srk
