// sr_dtw_dyn.cuh -- K2 (second form): the reference's greedy dtw (Src/Speech_Recog/DTW.C:120-192) with the (utterance,
// template) pairs handed to lanes DYNAMICALLY.
//
// The walk is sequential and its length depends on the data (somewhere between min(I, M) and I + M steps), so with a
// fixed lane = pair mapping a warp runs as long as its longest walk: ncu showed 21.9 of 32 lanes active per issued
// instruction in the static kernel (sr_dtw.cu). Here a CTA keeps its template tile (<= 32 templates) and a RING of
// staged utterances in shared memory; two producer warps stage utterances (byte planes + squared norms, as in
// sr_dtw.cu) into ring slots as they become free, and the 30 consumer warps pull pair numbers from one shared
// counter: whenever eight or more lanes of a warp are idle the warp claims new pairs for them (one warp-aggregated
// atomic), so lanes whose walk has ended do not wait for the longest walk of the warp. Slots are sized by the longest
// feature set actually present (max frm_num of the inputs, computed on the device by the caller; of the tile, computed
// here), not by vv_frm_max = 119: with ~35-frame utterances three times as many fit, which is what keeps > 2 pairs per
// lane staged ahead.
//
// Synchronisation is by monotonic counters in shared memory with release/acquire accesses:
//   flag[slot] = seq + 1   (producer, release)  -> the consumer that was handed a pair of utterance `seq` waits for it;
//   done[slot] += 1        (consumer, release, after its last read of the slot) -> the producer reuses the slot for
//                           utterance seq when done[slot] == (seq / R) * Tt.
// Rows, header decode, the tile stager, the walk step and the argmin epilogue are those of dtw_kernel (sr_dtw_core.cuh);
// results are identical. Included by sr_dtw.cu, whose launch_scan runs frm_max_kernel and then this kernel.
#pragma once
#include "sr_dtw_core.cuh"

namespace srk {

constexpr int kDynWarps = 32;
constexpr int kDynProducers = 2;
constexpr int kDynRMax = 192;               // ring slots the control arrays are sized for
constexpr int kDynRefill = 8;               // idle lanes of a warp that trigger a claim

__device__ __forceinline__ u32 ld_acquire_s(const u32 *p) {
    u32 v;
    asm volatile("ld.acquire.cta.shared.u32 %0, [%1];" : "=r"(v) : "r"(smem_u32(p)) : "memory");
    return v;
}
__device__ __forceinline__ void st_release_s(u32 *p, u32 v) {
    asm volatile("st.release.cta.shared.u32 [%0], %1;" ::"r"(smem_u32(p)), "r"(v) : "memory");
}
__device__ __forceinline__ void red_release_add_s(u32 *p, u32 v) {
    asm volatile("red.release.cta.shared.add.u32 [%0], %1;" ::"r"(smem_u32(p)), "r"(v) : "memory");
}

struct DynCtrl {
    u32 next_pair;
    u32 tmax;
    u32 pad[2];
    u32 tfrm[kTileT];
    u32 tslot_id[kTileT];
    u32 flag[kDynRMax];
    u32 done[kDynRMax];
    u32 ufrm[kDynRMax];
};

__host__ __device__ inline u32 dyn_slot_bytes(u32 rows) { return (rows * 28u + 7u) & ~7u; }

template <bool kLift>
__global__ void __launch_bounds__(kDynWarps * 32, 1)
dtw_dyn_kernel(const __grid_constant__ ScanArgs a, const unsigned char *__restrict__ in_ftr, const unsigned char *__restrict__ bank,
               const u8 *__restrict__ status, const u32 *__restrict__ B_dev, const u32 *__restrict__ perm,
               u32 *__restrict__ score, u64 *__restrict__ best, u32 tile0,
               u32 smem_bytes, const u32 *__restrict__ max_frm_dev /* max frm_num over the inputs, or NULL (assume 119) */) {
    extern __shared__ __align__(128) unsigned char smem_raw[];
    DynCtrl &c = *reinterpret_cast<DynCtrl *>(smem_raw);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    u32 B = a.B;
    if (B_dev) B = min(B, *B_dev);
    if (B == 0 || blockIdx.y >= B) return;
    const u32 t0 = (blockIdx.x + tile0) * kTileT;
    const int Tt = (int)min((u32)kTileT, a.T - t0);

    // ---- slot sizes from the longest template of the tile --------------------------------------------------------
    if (threadIdx.x == 0) { c.next_pair = 0; c.tmax = 0; }
    for (int i = threadIdx.x; i < kDynRMax; i += blockDim.x) { c.flag[i] = 0; c.done[i] = 0; }
    __syncthreads();
    if (threadIdx.x < Tt) {
        const u32 ts = perm ? perm[t0 + threadIdx.x] : t0 + threadIdx.x;
        const u32 frm = decode_frm(*reinterpret_cast<const u32 *>(bank + (size_t)ts * a.slot_stride), a.check_sign);
        if (frm != kNoWalk) atomicMax(&c.tmax, frm);
    }
    __syncthreads();
    const u32 trows = (u32)staged_rows(c.tmax);
    u32 umax = max_frm_dev ? *max_frm_dev : kMaxFrm;
    const u32 urows = (u32)staged_rows(min(umax, kMaxFrm));
    const u32 tslot = dyn_slot_bytes(trows), uslot = dyn_slot_bytes(urows);
    const u32 tnrm = trows * 24u, unrm = urows * 24u;
    unsigned char *tile = smem_raw + ((sizeof(DynCtrl) + 127) & ~127u);
    unsigned char *ring = tile + (((size_t)Tt * tslot + 127) & ~(size_t)127);
    const u32 ring_cap = smem_bytes - (u32)(ring - smem_raw);
    u32 R = ring_cap / uslot;
    if (R > (u32)kDynRMax) R = kDynRMax;

    stage_tile<kLift>(tile, tslot, tnrm, c.tfrm, c.tslot_id, bank, a.slot_stride, a.check_sign, perm, t0, Tt, warp, lane,
                      kDynWarps);
    __syncthreads();

    const u32 nseq = (B - blockIdx.y + gridDim.y - 1) / gridDim.y;       // utterances of this CTA: blockIdx.y + seq*gridDim.y
    const u32 total_pairs = nseq * (u32)Tt;

    if (warp < kDynProducers) {
        // ============================ producers: stage utterances into free ring slots ===========================
        for (u32 seq = warp; seq < nseq; seq += kDynProducers) {
            const u32 slot = seq % R;
            const u32 want = (seq / R) * (u32)Tt;                        // pairs completed on this slot before it is reused
            if (lane == 0) while (ld_acquire_s(&c.done[slot]) != want) __nanosleep(64);
            __syncwarp();
            const u32 u = blockIdx.y + seq * gridDim.y;
            u32 frm = kNoWalk;
            if (!(status && status[u] != SR_ST_OK)) {                    // VAD/MFCC failed: spch_recg returns before dtw
                const unsigned char *uf = in_ftr + (size_t)u * kFtrBytes;
                frm = decode_frm(*reinterpret_cast<const u32 *>(uf), false);
                stage_planes<kLift>(ring + (size_t)slot * uslot, unrm, uf, min(staged_rows(frm), (int)urows), lane, 32);
            }
            __syncwarp();
            if (lane == 0) { c.ufrm[slot] = frm; st_release_s(&c.flag[slot], seq + 1u); }
        }
        return;
    }

    // ================================ consumers: pull pairs, walk ===================================================
    bool active = false, exhausted = false;
    PRow i0, i1, m0, m1;
    const unsigned char *urow = ring, *trow = tile;   // shared from the start: kept as 32-bit shared addresses
    u32 dis = 0, step = 0, slot = 0, out_u = 0, out_t = 0;
    int x = 0, y = 0, I = 0, M = 0, X1 = 0, X2 = 0, ya0 = 0, yb0 = 0, ya1 = 0, yb1 = 0;
    auto finish = [&](u32 result) {
        emit_pair(score, best, a, out_u, out_t, result);
        red_release_add_s(&c.done[slot], 1u);
        active = false;
    };

    // A lane never blocks inside the warp: a claimed pair whose utterance is not staged yet leaves the lane PENDING and the
    // flag is polled once per loop iteration while the warp's other lanes keep walking. (A spin inside the divergent claim
    // path could wait for a ring slot whose previous occupant is still being walked by a lane of the SAME warp, parked at
    // the reconvergence point: deadlock.)
    bool pending = false;
    u32 pend_seq = 0, pend_tl = 0;
    for (;;) {
        const u32 act = __ballot_sync(0xFFFFFFFFu, active);
        const u32 pnd = __ballot_sync(0xFFFFFFFFu, pending);
        const u32 idle = __ballot_sync(0xFFFFFFFFu, !active && !pending && !exhausted);
        if (idle && ((act | pnd) == 0 || __popc(idle) >= kDynRefill)) {
            u32 base = 0;
            const int leader = __ffs(idle) - 1;
            if (lane == leader) base = atomicAdd(&c.next_pair, (u32)__popc(idle));
            base = __shfl_sync(0xFFFFFFFFu, base, leader);
            if (!active && !pending && !exhausted) {
                const u32 p = base + (u32)__popc(idle & ((1u << lane) - 1u));
                if (p >= total_pairs) exhausted = true;
                else { pend_seq = p / (u32)Tt; pend_tl = p - pend_seq * (u32)Tt; pending = true; }
            }
        } else if ((act | pnd | idle) == 0) break;                        // every lane has run out of pairs
        if (pending) {
            slot = pend_seq % R;
            if (ld_acquire_s(&c.flag[slot]) == pend_seq + 1u) {           // staged: start the walk (or reject at once)
                pending = false;
                out_u = blockIdx.y + pend_seq * gridDim.y; out_t = c.tslot_id[pend_tl];
                const u32 Iraw = c.ufrm[slot], Mraw = c.tfrm[pend_tl];
                if (!pair_walks(Iraw, Mraw, true)) finish(SR_DIS_ERR);
                else {
                    urow = ring + slot * uslot; trow = tile + pend_tl * tslot;
                    I = (int)Iraw; M = (int)Mraw;
                    greedy_start(I, M, X1, X2, i0, i1, m0, m1, dis, step, x, y, ya0, yb0, ya1, yb1, urow, unrm, trow, tnrm);
                    active = true;
                }
            } else if (act == 0) __nanosleep(100);                        // nothing to walk meanwhile: do not hammer the flag
        } else if (active) {
            if (!greedy_step(I, M, X1, X2, i0, i1, m0, m1, dis, step, x, y, ya0, yb0, ya1, yb1, urow, unrm, trow, tnrm))
                finish(dis / (step & 0xFFFFu));                           // DTW.C:191 (step is u16)
        }
    }
}

// max frm_num (<= 119) over B feature sets -> *out (device); `status` gates like the kernel does
__global__ void frm_max_kernel(const unsigned char *__restrict__ ftr, u32 B, const u8 *__restrict__ status, u32 *out,
                               const u32 *__restrict__ B_dev) {
    if (B_dev) B = min(B, *B_dev);
    u32 m = 0;
    for (u32 i = blockIdx.x * blockDim.x + threadIdx.x; i < B; i += gridDim.x * blockDim.x) {
        if (status && status[i] != SR_ST_OK) continue;
        const u32 f = (*reinterpret_cast<const u32 *>(ftr + (size_t)i * kFtrBytes)) >> 16;
        if (f <= 119u) m = max(m, f);
    }
#pragma unroll
    for (int o = 16; o; o >>= 1) m = max(m, __shfl_xor_sync(0xFFFFFFFFu, m, o));
    if ((threadIdx.x & 31) == 0 && m) atomicMax(out, m);
}

}  // namespace srk
