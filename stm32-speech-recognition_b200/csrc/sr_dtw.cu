// sr_dtw.cu -- K2: batched dtw (Src/Speech_Recog/DTW.C:120-192) = the reference's GREEDY walk through
// the slope-2 / slope-1/2 parallelogram (dtw_limit, DTW.C:76-109) with the 12-dim integer local
// distance get_dis (DTW.C:45-62), plus the spch_recg argmin (Src/APP/main.c:276-291) as an epilogue.
//
// Mapping: one thread per (utterance, template) pair -- the walk is inherently sequential and data
// dependent; parallelism is across the B x T pairs. A CTA keeps a tile of up to 32 templates in shared
// memory (loaded once, reused for every utterance the CTA visits). Its 32 warps are split into groups
// of Wg warps; a group stages NU utterances at a time and its 32*Wg lanes walk the NU x Tt pairs
// (flattened), so lanes stay busy when Tt < 32 (the host picks NU/Wg for the tile width).
// dtw_limit is evaluated as a per-column y interval (ya, yb) updated only when x moves. Rows, header decode, the walk and
// the epilogue are the shared core of sr_dtw_core.cuh.
// Every template-scan kernel takes one ScanArgs; scan_plan and launch_scan at the end of this file are the one place the
// matcher flags are decoded and a matcher becomes a kernel launch.
#include "sr_internal.h"
#include "sr_dtw_dyn.cuh"

namespace srk {

constexpr int kDtwWarps = 16;
constexpr int kK2Warps = 32;                // lane-packed kernels: 1024 threads x 64 registers, more walks in flight per SM
constexpr int kTileHdr = 256;               // after the tile: [32] frame counts, then [32] bank slot numbers

__device__ __forceinline__ void group_barrier(int id, int nthreads) {
    if (nthreads == 32) __syncwarp();
    else asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}

// The lane-packed tile scan of dtw_kernel and dtw_band_thread_kernel. A CTA stages a tile of Tt <= 32 templates; its
// warps, in G groups of Wg, stage NU utterances at a time, and each lane of a group scores one fixed (utterance slot,
// template) pair of the NU x Tt (flattened), so lanes stay busy when Tt < 32. pair(I, M, urow, trow) scores a pair
// that passed pair_walks(guard). kLift: inputs and templates staged liftered (SR_DTW_LIFTER). tslots: template slots
// allocated in shared memory. The pointers are the kernel's (SCAN_PTRS).
template <bool kLift, class Pair>
__device__ __forceinline__ void lane_packed_scan(const ScanArgs &a, const unsigned char *in_ftr, const unsigned char *bank,
                                                 const u8 *status, const u32 *B_dev, const u32 *perm, u32 *score, u64 *best,
                                                 int Wg, int NU, int G, u32 tile0, int tslots, bool guard, Pair pair) {
    extern __shared__ __align__(128) unsigned char smem_raw[];
    u32 B = a.B;
    if (B_dev) B = min(B, *B_dev);
    if (B == 0) return;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const u32 t0 = (blockIdx.x + tile0) * kTileT;
    const int Tt = (int)min((u32)kTileT, a.T - t0);
    unsigned char *tile = smem_raw;                                                // Tt slots
    u32 *tfrm = reinterpret_cast<u32 *>(smem_raw + (size_t)tslots * kSlotBytes);
    unsigned char *uslots = smem_raw + (size_t)tslots * kSlotBytes + kTileHdr;     // G*NU slots
    u32 *ufrm = reinterpret_cast<u32 *>(uslots + (size_t)G * NU * kSlotBytes);     // [G*NU]

    stage_tile<kLift>(tile, kSlotBytes, kNrm119, tfrm, tfrm + kTileT, bank, a.slot_stride, a.check_sign, perm, t0, Tt, warp,
                      lane, kK2Warps);
    __syncthreads();

    const int group = warp / Wg, wig = warp - group * Wg;
    if (group >= G) return;                                            // idle warps (32 not divisible by Wg)
    const int gthreads = Wg * 32, gtid = wig * 32 + lane;
    const int ul = gtid / Tt, tl = gtid - ul * Tt;                     // this lane's (utterance slot, template) -- fixed
    const bool lane_has_pair = ul < NU;
    unsigned char *gslots = uslots + (size_t)group * NU * kSlotBytes;
    u32 *gfrm = ufrm + group * NU;
    const unsigned char *trow = tile + (size_t)tl * kSlotBytes;
    const u32 Mraw = lane_has_pair ? tfrm[tl] : kNoWalk;

    for (u32 ubase = (blockIdx.y * G + group) * NU; ubase < B; ubase += gridDim.y * G * NU) {
        // ---- stage NU utterances of this group ---------------------------------------------------------
        for (int s = 0; s < NU; ++s) {
            const u32 u = ubase + s;
            u32 frm = kNoWalk;
            if (u < B && !(status && status[u] != SR_ST_OK)) {        // VAD/MFCC failed: spch_recg returns before dtw
                const unsigned char *uf = in_ftr + (size_t)u * kFtrBytes;
                frm = decode_frm(*reinterpret_cast<const u32 *>(uf), false);
                stage_planes<kLift>(gslots + (size_t)s * kSlotBytes, kNrm119, uf, staged_rows(frm), gtid, gthreads);
            }
            if (gtid == 0) gfrm[s] = frm;
        }
        group_barrier(1 + group, gthreads);

        const u32 u = ubase + (u32)ul;
        if (lane_has_pair && u < B) {
            const u32 Iraw = gfrm[ul];
            const u32 result = pair_walks(Iraw, Mraw, guard) ? pair((int)Iraw, (int)Mraw, gslots + (size_t)ul * kSlotBytes, trow)
                                                      : SR_DIS_ERR;
            const u32 t = perm ? tfrm[kTileT + tl] : t0 + (u32)tl;   // the original slot number: score column, argmin key
            emit_pair(score, best, a, u, t, result);
        }
        group_barrier(1 + group, gthreads);                                                          // before restaging
    }
}

template <bool kLift>
__global__ void __launch_bounds__(kK2Warps * 32)
dtw_kernel(const __grid_constant__ ScanArgs a, const unsigned char *__restrict__ in_ftr, const unsigned char *__restrict__ bank,
           const u8 *__restrict__ status, const u32 *__restrict__ B_dev, const u32 *__restrict__ perm,
           u32 *__restrict__ score, u64 *__restrict__ best, int Wg, int NU, int G, u32 tile0,
           int tslots) {
    lane_packed_scan<kLift>(a, in_ftr, bank, status, B_dev, perm, score, best, Wg, NU, G, tile0, tslots, true,
                            [](int I, int M, const unsigned char *urow, const unsigned char *trow) {
                         PRow i0, i1, m0, m1;
                         u32 dis, steps;
                         int X1, X2, x, y, ya0, yb0, ya1, yb1;
                         greedy_start(I, M, X1, X2, i0, i1, m0, m1, dis, steps, x, y, ya0, yb0, ya1, yb1, urow, kNrm119, trow,
                                      kNrm119);
                         while (greedy_step(I, M, X1, X2, i0, i1, m0, m1, dis, steps, x, y, ya0, yb0, ya1, yb1, urow, kNrm119,
                                            trow, kNrm119)) {}
                         return dis / (steps & 0xFFFFu);                                         // DTW.C:191 (step is u16)
                     });
}

// best[] initialiser and finaliser (main.c:276-278 min_comm=0, min_dis=dis_max; main.c:292-294)
__global__ void best_init_kernel(u64 *best, u32 B) {
    const u32 i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < B) best[i] = kKeyStart;
}
// The decision of each of B utterances (decide) into the fields NULL does not mark as unwanted (NULL status: every
// utterance OK). Without a rule the keys are best's; under one (kRule) they are rows of C keys (ScanArgs), and the
// decision's key goes to best[i] (what an all-gather reads) and SR_ST_REJECT into status. The rule comes last.
template <bool kRule>
__global__ void best_final_kernel(const u64 *keys, u32 B, u32 *best_idx, u32 *best_dis, u32 *cmd, u8 *status, u64 *best,
                                  Rule rl) {
    const u32 g = kRule ? rule_lanes(rl) : 1u;
    const u32 i = (blockIdx.x * blockDim.x + threadIdx.x) / g;
    if (i >= B) return;                                                         // whole warps: B * g threads
    const u32 st = status ? status[i] : SR_ST_OK;
    Decision d;
    if (!decide<kRule>(keys, i, st, rl, g, d)) return;
    if constexpr (kRule) {
        best[i] = d.key;
        if (d.status != st) status[i] = (u8)d.status;
    }
    if (best_idx) best_idx[i] = d.idx;
    if (best_dis) best_dis[i] = d.dis;
    if (cmd) cmd[i] = d.cmd;
}

// status of the recognise pipeline from VAD/MFCC results (main.c:261-274)
__global__ void status_kernel(const u32 *seg_off, const unsigned char *ftr, u32 B, u8 *status) {
    const u32 i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= B) return;
    u8 st = SR_ST_OK;
    if (seg_off[(size_t)i * 6 + 1] == SR_SEG_NULL) st = SR_ST_VAD_FAIL;
    else if (((*reinterpret_cast<const u32 *>(ftr + (size_t)i * kFtrBytes)) >> 16) == 0) st = SR_ST_MFCC_FAIL;
    status[i] = st;
}

// exhaustive self-check of sqrt_rn_normal against the IEEE intrinsic over float bit patterns [lo, hi)
__global__ void sqrt_check_kernel(u32 lo, u32 hi, unsigned long long *bad) {
    unsigned long long n = 0;
    for (u64 b = (u64)lo + blockIdx.x * (u64)blockDim.x + threadIdx.x; b < hi; b += (u64)gridDim.x * blockDim.x) {
        const float x = __uint_as_float((u32)b);
        if (__float_as_uint(sqrt_rn_normal(x)) != __float_as_uint(__fsqrt_rn(x))) ++n;
    }
    if (n) atomicAdd(bad, n);
}
cudaError_t launch_sqrt_check(u32 lo, u32 hi, unsigned long long *bad_dev, cudaStream_t st) {
    sqrt_check_kernel<<<132 * 8, 256, 0, st>>>(lo, hi, bad_dev);
    return cudaGetLastError();
}

// ---- get_mdl / get_mean (DTW.C:195-296): the reference's (never called) template averaging ----------------
// Same greedy walk as dtw() between two feature sets; every visited point (x,y) emits the element-wise mean
// (a+b)/2 (C truncation, DTW.C:201) of in1[x-1] and in2[y-1] as the next row of the model; frm_num = number of
// points, return value dis/step. One thread per pair (not a hot path). The reference writes past mfcc_dat when
// the path is longer than vv_frm_max rows; here rows beyond 118 are dropped and frm_num is clamped to 119.
__device__ __forceinline__ u32 get_dis_rows(const s16 *a, const s16 *b) {
    u32 d = 0;
#pragma unroll
    for (int j = 0; j < 12; ++j) { const s32 dif = (s32)a[j] - (s32)b[j]; d += (u32)dif * (u32)dif; }
    return usqrt_trunc(d);
}
__device__ __forceinline__ bool ins_xy(int x, int y, int X1, int X2, int I, int M) {
    const bool out_a = (x < X1) ? (y >= 2 * x + 2) : (2 * y + I - 2 * M >= x + 4);
    const bool out_b = (x < X2) ? (2 * y + 2 <= x) : (y + 4 <= 2 * x + M - 2 * I);
    return !(out_a || out_b);
}
__global__ void get_mdl_kernel(const unsigned char *in1, const unsigned char *in2, unsigned char *mdl, u32 n, u32 *dis_out) {
    const u32 p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= n) return;
    const unsigned char *f1 = in1 + (size_t)p * kFtrBytes, *f2 = in2 + (size_t)p * kFtrBytes;
    unsigned char *fm = mdl + (size_t)p * kFtrBytes;
    const int I = (int)(*reinterpret_cast<const u16 *>(f1 + 2)), M = (int)(*reinterpret_cast<const u16 *>(f2 + 2));
    if (I > M * 2 || 2 * I < M || I > 119 || M > 119) { dis_out[p] = SR_DIS_ERR; return; }      // DTW.C:231-234: mdl untouched
    const s16 *a = reinterpret_cast<const s16 *>(f1 + 4), *b = reinterpret_cast<const s16 *>(f2 + 4);
    s16 *m = reinterpret_cast<s16 *>(fm + 4);
    const int X1 = (2 * M - I) / 3, X2 = (4 * I - 2 * M) / 3;
    auto mean_row = [&](int row, const s16 *ra, const s16 *rb) {
        if (row >= 119) return;
        for (int j = 0; j < 12; ++j) m[row * 12 + j] = (s16)(((s32)ra[j] + (s32)rb[j]) / 2);
    };
    u32 dis = get_dis_rows(a, b);
    mean_row(0, a, b);
    int x = 1, y = 1;
    u32 step = 1;
    do {
        const u32 up = ins_xy(x, y + 1, X1, X2, I, M) ? get_dis_rows(b + 12 * y, a + 12 * (x - 1)) : SR_DIS_ERR;
        const u32 right = ins_xy(x + 1, y, X1, X2, I, M) ? get_dis_rows(b + 12 * (y - 1), a + 12 * x) : SR_DIS_ERR;
        const u32 ru = ins_xy(x + 1, y + 1, X1, X2, I, M) ? get_dis_rows(b + 12 * y, a + 12 * x) : SR_DIS_ERR;
        u32 mn = ru;
        if (mn > right) mn = right;
        if (mn > up) mn = up;
        dis += mn;
        if (mn == ru) { ++x; ++y; } else if (mn == up) { ++y; } else { ++x; }
        mean_row((int)step, a + 12 * (x - 1), b + 12 * (y - 1));                                   // DTW.C:286-287
        ++step;
    } while (x < I && y < M);
    *reinterpret_cast<u16 *>(fm + 2) = (u16)min(step, 119u);                                         // DTW.C:293
    dis_out[p] = dis / step;
}

// ---- save_ftr_mdl (Flash.C:17-67) for a batch: flash-layout slots from freshly computed features -------------
__global__ void pack_slots_kernel(const unsigned char *ftr, const u8 *status, u32 B, unsigned char *bank, u32 slot_stride) {
    const u32 b = blockIdx.x;
    if (b >= B) return;
    u32 *dst = reinterpret_cast<u32 *>(bank + (size_t)b * slot_stride);
    const u32 *src = reinterpret_cast<const u32 *>(ftr + (size_t)b * kFtrBytes);
    const bool ok = status[b] == SR_ST_OK;
    const u32 frm = src[0] >> 16;
    const u32 used = ok ? 1u + 6u * frm : 0u;                      // header word + 6 words per row (Flash.C:27,56-63)
    for (u32 i = threadIdx.x; i < slot_stride / 4; i += blockDim.x) {
        u32 v = 0xFFFFFFFFu;                                       // erased flash (Flash.C:32-39)
        if (i < used) v = i == 0 ? ((frm << 16) | SR_SAVE_MASK) : src[i];
        dst[i] = v;
    }
}
cudaError_t launch_get_mdl(const void *in1, const void *in2, void *mdl, u32 n, u32 *dis, cudaStream_t st) {
    if (n == 0) return cudaSuccess;
    get_mdl_kernel<<<(n + 63) / 64, 64, 0, st>>>(static_cast<const unsigned char *>(in1), static_cast<const unsigned char *>(in2),
                                                static_cast<unsigned char *>(mdl), n, dis);
    return cudaGetLastError();
}
cudaError_t launch_pack_slots(const void *ftr, const u8 *status, u32 B, void *bank, u32 slot_stride, cudaStream_t st) {
    if (B == 0) return cudaSuccess;
    pack_slots_kernel<<<B, 128, 0, st>>>(static_cast<const unsigned char *>(ftr), status, B, static_cast<unsigned char *>(bank), slot_stride);
    return cudaGetLastError();
}

// dtw_limit (DTW.C:76-109) for n points: out[i] = 0 "ins" / 1 "outs" for (x[i], y[i]) in the parallelogram of (I[i], M[i])
__global__ void dtw_limit_kernel(const u16 *x, const u16 *y, const u16 *I, const u16 *M, u32 n, u8 *out) {
    const u32 i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int Ii = I[i], Mi = M[i];
    const int X1 = (int)(u16)((2 * Mi - Ii) / 3), X2 = (int)(u16)((4 * Ii - 2 * Mi) / 3);   // u16 statics, DTW.C:65-66,141-142
    out[i] = ins_xy(x[i], y[i], X1, X2, Ii, Mi) ? 0 : 1;
}
cudaError_t launch_dtw_limit(const u16 *x, const u16 *y, const u16 *I, const u16 *M, u32 n, u8 *out, cudaStream_t st) {
    if (n == 0) return cudaSuccess;
    dtw_limit_kernel<<<(n + 255) / 256, 256, 0, st>>>(x, y, I, M, n, out);
    return cudaGetLastError();
}

// get_dis for n independent row pairs (secondary drop-in symbol, DTW.C:45-62)
__global__ void get_dis_kernel(const s16 *a, const s16 *b, u32 n, u32 *out) {
    const u32 i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    out[i] = get_dis_rows(a + (size_t)i * 12, b + (size_t)i * 12);
}

// lane packing of a tile of width Tt for lane_packed_scan: groups of Wg warps walk NU utterances x Tt templates; the
// (Wg, NU, G) with the most busy lanes, and the shared memory it takes
struct LanePlan { int Wg, NU, G; size_t smem; };
static LanePlan plan_lanes(int Tt) {
    constexpr int kSmemMax = 224 * 1024;
    const size_t budget = kSmemMax - (size_t)Tt * kSlotBytes - kTileHdr - 512;
    const int slots_max = (int)(budget / kSlotBytes);
    LanePlan p{1, 1, 1, 0};
    double best_util = -1.0;
    for (int Wg = 1; Wg <= 8; ++Wg) {
        const int NU = (32 * Wg) / Tt;
        if (NU < 1) continue;
        int G = kK2Warps / Wg;
        if (G > slots_max / NU) G = slots_max / NU;
        if (Wg > 1 && G > 15) G = 15;                       // named barriers 1..15
        if (G < 1) continue;
        const double util = ((double)NU * Tt / (32.0 * Wg)) * ((double)G * Wg / kK2Warps);
        if (util > best_util + 1e-9) { best_util = util; p.Wg = Wg; p.NU = NU; p.G = G; }
    }
    p.smem = (size_t)Tt * kSlotBytes + kTileHdr + (size_t)p.G * p.NU * kSlotBytes + (size_t)p.G * p.NU * 4 + 64;
    return p;
}

cudaError_t launch_best_init(u64 *best, u64 n, cudaStream_t st) {
    if (n == 0) return cudaSuccess;
    if (n > 0xFFFFFF00ull) return cudaErrorInvalidValue;            // 32 GB of keys: past any workspace anyway
    best_init_kernel<<<(u32)((n + 255) / 256), 256, 0, st>>>(best, (u32)n);
    return cudaGetLastError();
}
cudaError_t launch_best_final(u64 *best, const u64 *keys, u32 B, const Rule &rl, u32 *best_idx, u32 *best_dis, u32 *cmd,
                              u8 *status, cudaStream_t st) {
    if (B == 0) return cudaSuccess;
    (rl.C ? best_final_kernel<true> : best_final_kernel<false>)<<<rule_grid(B, rl), 256, 0, st>>>(
        keys, B, best_idx, best_dis, cmd, status, best, rl);
    return cudaGetLastError();
}
cudaError_t launch_status(const u32 *seg_off, const void *ftr, u32 B, u8 *status, cudaStream_t st) {
    if (B == 0) return cudaSuccess;
    status_kernel<<<(B + 255) / 256, 256, 0, st>>>(seg_off, static_cast<const unsigned char *>(ftr), B, status);
    return cudaGetLastError();
}
cudaError_t launch_get_dis(const s16 *a, const s16 *b, u32 n, u32 *out, cudaStream_t st) {
    if (n == 0) return cudaSuccess;
    get_dis_kernel<<<(n + 255) / 256, 256, 0, st>>>(a, b, n, out);
    return cudaGetLastError();
}

}  // namespace srk

// ---- K3: Sakoe-Chiba banded DP (EXTENSION: not in the reference, whose dtw() is the greedy walk above;
// BASELINE.json configs[2] names it; checked against our own CPU DP oracle sro_dtw_band -- parity unpinned
// by the reference). D(i,j) = d(i,j) + min(D(i-1,j), D(i,j-1), D(i-1,j-1)), band |j - floor(i*M/I)| <= r,
// local distance = get_dis, result D(I-1,M-1)/(I+M), same 2:1 length guard as DTW.C:133 unless the plan turns it off
// (SR_DTW_ANY_RATE). Without the guard the band centre c = floor(i*M/I) moves by up to 118 columns per row (M > 2I), not
// 0..2, and stays put for several rows when M < I/2; every kernel below takes any shift, and a shift past 2r + 1 leaves
// the new row unreachable.
// Three kernels, chosen from r alone (launch_scan): dtw_band_thread_kernel<10> for r = 10, dtw_band_kernel for the
// other r <= 15, dtw_wide_kernel for r >= 16 up to the full matrix. On the recognition path all three take the
// per-utterance status gate, a batch size produced on the device (streaming) and the bank order; scores and argmin keys
// stay under the original slot number.
// dtw_band_kernel: one WARP per (utterance, template) cost matrix, lane = band offset (2r+1 <= 32). The in-row dependency
// x_j = d_j + min(A_j, x_{j-1}) is a (min,+) linear recurrence, solved per row with two warp scans:
//   P = prefix-sum(d),  x_j = P_j + prefix-min_k( A_k - P_{k-1} );  A comes from the previous row by shuffles.
namespace srk {

constexpr s32 kInf = 0x3FFFFFFF;

// The warp-per-pair tile scan of dtw_band_kernel and dtw_wide_kernel. A CTA stages a tile of Tt <= 32 templates (bank
// slot perm[t] when a bank order is given); each warp stages one utterance at a time and scores it against the Tt
// templates one after another, the whole warp on one cost matrix: pair(I, M, urow, trow, lane) returns, in every lane, the
// score of a pair that passed pair_walks(guard). Lane tt keeps the score of template tt; one score row and one atomicMin
// of the warp's smallest key per utterance (under a decision rule, one per lane into its key of the row). An utterance
// whose status is not SR_ST_OK scores SR_DIS_ERR, as in
// lane_packed_scan. kLift: inputs and templates staged liftered (SR_DTW_LIFTER).
template <bool kLift, class Pair>
__device__ __forceinline__ void warp_pair_scan(const ScanArgs &a, const unsigned char *in_ftr, const unsigned char *bank,
                                               const u8 *status, const u32 *B_dev, const u32 *perm, u32 *score, u64 *best,
                                               bool guard, Pair pair) {
    extern __shared__ __align__(128) unsigned char smem_raw[];
    u32 B = a.B;
    if (B_dev) B = min(B, *B_dev);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const u32 t0 = blockIdx.x * kTileT;
    const int Tt = (int)min((u32)kTileT, a.T - t0);
    unsigned char *tile = smem_raw;                                               // byte-plane slots, as in dtw_kernel
    u32 *tfrm = reinterpret_cast<u32 *>(smem_raw + (size_t)kTileT * kSlotBytes);  // [32] frame counts, [32] slot numbers
    unsigned char *uslot = smem_raw + (size_t)kTileT * kSlotBytes + kTileHdr + (size_t)warp * kSlotBytes;
    stage_tile<kLift>(tile, kSlotBytes, kNrm119, tfrm, tfrm + kTileT, bank, a.slot_stride, a.check_sign, perm, t0, Tt, warp,
                      lane, kDtwWarps);
    __syncthreads();
    for (u32 u = blockIdx.y * kDtwWarps + warp; u < B; u += gridDim.y * kDtwWarps) {
        const unsigned char *uf = in_ftr + (size_t)u * kFtrBytes;
        u32 Iraw = kNoWalk;                               // VAD/MFCC failed: spch_recg returns before dtw
        if (!(status && status[u] != SR_ST_OK)) Iraw = decode_frm(*reinterpret_cast<const u32 *>(uf), false);
        __syncwarp();
        stage_planes<kLift>(uslot, kNrm119, uf, staged_rows(Iraw), lane, 32);
        __syncwarp();
        u32 my_result = SR_DIS_ERR;                       // lane tt keeps the result of template tt
        for (int tt = 0; tt < Tt; ++tt) {
            const u32 Mraw = tfrm[tt];
            u32 result = SR_DIS_ERR;
            if (Iraw >= 1 && pair_walks(Iraw, Mraw, guard))
                result = pair((int)Iraw, (int)Mraw, uslot, tile + (size_t)tt * kSlotBytes, lane);
            if (lane == tt) my_result = result;
        }
        const bool has_t = lane < Tt;
        const u32 t = !has_t ? 0u : perm ? tfrm[kTileT + lane] : t0 + (u32)lane;   // the original slot number
        if (has_t && score) score[(size_t)u * a.T + t] = my_result;
        if (best && key_rows(a)) {                         // a decision rule: each lane its own key of the row
            if (has_t) atomicMin(reinterpret_cast<unsigned long long *>(key_of(best, a, u, t)),
                                 (unsigned long long)(((u64)my_result << 32) | (u64)t));
        } else if (best) {
            u64 key = has_t ? (((u64)my_result << 32) | (u64)t) : ~0ull;
#pragma unroll
            for (int o = 16; o; o >>= 1) { const u64 other = __shfl_xor_sync(0xFFFFFFFFu, key, o); key = other < key ? other : key; }
            if (lane == 0) atomicMin(reinterpret_cast<unsigned long long *>(&best[u]), (unsigned long long)key);
        }
    }
}

template <bool kLift>
__global__ void __launch_bounds__(kDtwWarps * 32)
dtw_band_kernel(const __grid_constant__ ScanArgs a, const unsigned char *__restrict__ in_ftr, const unsigned char *__restrict__ bank,
                const u8 *__restrict__ status, const u32 *__restrict__ B_dev, const u32 *__restrict__ perm,
                u32 *__restrict__ score, u64 *__restrict__ best) {
    // the previous row's cell of column j sits in lane j - (cprev - r): up and diag come from lanes lane + sft and
    // lane + sft - 1, and any lane past 31 or past 2r (those hold kInf) is out of the previous row's band, whatever sft is
    warp_pair_scan<kLift>(a, in_ftr, bank, status, B_dev, perm, score, best, a.guard,
                          [r = a.r](int I, int M, const unsigned char *uslot, const unsigned char *trow, int lane) {
        s32 Dprev = kInf;
        int cprev = 0;
        for (int i = 0; i < I; ++i) {
            const int c = (i * M) / I, j = c - r + lane;
            const bool valid = lane <= 2 * r && j >= 0 && j < M;
            PRow a, b;
            load_row(a, uslot, kNrm119, i);                            // broadcast read
            load_row(b, trow, kNrm119, valid ? j : 0);
            const s32 d = valid ? (s32)pdist(a, b) : 0;
            const int sft = c - cprev;
            const int su = lane + sft, sd = lane + sft - 1;
            s32 up = __shfl_sync(0xFFFFFFFFu, Dprev, su & 31);
            s32 dg = __shfl_sync(0xFFFFFFFFu, Dprev, sd & 31);
            if (su > 31) up = kInf;
            if (sd < 0 || sd > 31) dg = kInf;
            s32 A = min(up, dg);
            if (i == 0) A = (j == 0) ? 0 : kInf;
            if (!valid) A = kInf;
            s32 P = d;                                                 // inclusive prefix sum over lanes
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) { const s32 v = __shfl_up_sync(0xFFFFFFFFu, P, o); if (lane >= o) P += v; }
            s32 m = A - (P - d);                                       // A_k - P_{k-1}
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) { const s32 v = __shfl_up_sync(0xFFFFFFFFu, m, o); if (lane >= o) m = min(m, v); }
            s32 x = P + m;
            if (!valid || x >= kInf / 2) x = kInf;
            Dprev = x;
            cprev = c;
        }
        const int lend = (M - 1) - (cprev - r);                        // lane holding column M-1 in the last row
        const s32 fin = __shfl_sync(0xFFFFFFFFu, Dprev, lend & 31);
        return (lend >= 0 && lend <= 2 * r && fin < kInf / 2) ? (u32)fin / (u32)(I + M) : SR_DIS_ERR;
    });
}

// ---- K3w: the same DP for r >= 16 up to the full matrix: one WARP per pair, a whole ROW across the warp ---------------
// A row never has more than M <= 119 valid columns, whatever r is, so lane l holds the fixed columns 4l .. 4l+3 (32 x 4 =
// 128 >= 119) and the cost of a pair does not depend on r: r >= 118 is the unconstrained DTW (the host clamps r to 118).
// The band of row i is the column interval [max(c-r, 0), min(c+r, M-1)], c = floor(i*M/I); cells outside it are +inf.
// Each row is one dp_column step (sr_dtw_core.cuh, which also gives the headroom of kInf); the template's four rows
// stay in registers for the whole pair.
template <bool kLift>
__global__ void __launch_bounds__(kDtwWarps * 32, 1)       // one CTA per SM (shared memory): up to 128 registers
dtw_wide_kernel(const __grid_constant__ ScanArgs a, const unsigned char *__restrict__ in_ftr, const unsigned char *__restrict__ bank,
                const u8 *__restrict__ status, const u32 *__restrict__ B_dev, const u32 *__restrict__ perm,
                u32 *__restrict__ score, u64 *__restrict__ best) {
    warp_pair_scan<kLift>(a, in_ftr, bank, status, B_dev, perm, score, best, a.guard,
                          [r = a.r](int I, int M, const unsigned char *uslot, const unsigned char *trow, int lane) {
        const int j0 = lane * 4;
        PRow b[4];
        s32 D[4];
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            load_row(b[k], trow, kNrm119, j0 + k < M ? j0 + k : 0);
            D[k] = kInf;
        }
        for (int i = 0; i < I; ++i) {
            const int c = (i * M) / I, lo = max(c - r, 0), hi = min(c + r, M - 1);
            PRow a;
            load_row(a, uslot, kNrm119, i);                            // broadcast read
            dp_column<s32, kInf>(D, lane, [&](int k, s32 up, s32 dg, s32 &d, s32 &A, bool &valid) {
                const int j = j0 + k;
                valid = j >= lo && j <= hi;
                d = valid ? (s32)pdist(a, b[k]) : 0;
                A = i == 0 ? (j == 0 ? 0 : kInf) : min(up, dg);
            }, [](int, s32, s32) {});
        }
        const s32 fin = dp_end(D, (M - 1) & 3, (M - 1) / 4);
        return fin < kInf / 2 ? (u32)fin / (u32)(I + M) : SR_DIS_ERR;
    });
}

// ---- K3b: the same banded DP, one THREAD per pair, band in registers (compile-time radius) -----------------------
// 3.7x fewer issue slots per lattice cell than the warp-scan form: no scans, no idle lanes (21 of 32), and the
// lane-packed tile scan of dtw_kernel. The band of row i sits at columns c_i-R..c_i+R with
// c_i = floor(i*M/I); it slides by s = c_i - c_{i-1} in {0,1,2} per row under the 2:1 guard, realised as two
// predicated shift-by-one passes over the register array (no divergence between lanes whose templates have different
// lengths). Under SR_DTW_ANY_RATE a row may slide further (M > 2I): those rows take a loop of min(s, W) - 2 more passes
// after the two, so the passes of a pair total at most M - 1, and a slide past W leaves no cell of the old row.
template <int R, bool kLift>
__global__ void __launch_bounds__(kK2Warps * 32)
dtw_band_thread_kernel(const __grid_constant__ ScanArgs a, const unsigned char *__restrict__ in_ftr, const unsigned char *__restrict__ bank,
                       const u8 *__restrict__ status, const u32 *__restrict__ B_dev, const u32 *__restrict__ perm,
                       u32 *__restrict__ score, u64 *__restrict__ best, int Wg, int NU,
                       int G, u32 tile0, int tslots) {
    lane_packed_scan<kLift>(a, in_ftr, bank, status, B_dev, perm, score, best, Wg, NU, G, tile0, tslots, a.guard,
                            [](int I, int M, const unsigned char *urow, const unsigned char *trow) {
        constexpr int W = 2 * R + 1;
        if (I == 0 || M == 0) return SR_DIS_ERR;           // empty feature sets: no cell
        s32 D[W];
#pragma unroll
        for (int k = 0; k < W; ++k) D[k] = kInf;
        int c = 0, cprev = 0, err = 0;                     // c = floor(i*M/I) kept incrementally: i*M = c*I + err
        for (int i = 0; i < I; ++i) {
            const int sft = c - cprev;                     // 0, 1 or 2 when M <= 2I; up to M - 1 otherwise
            // diag source of cell k=0 is the old element at index sft-1
            s32 dm1 = sft == 2 ? D[1] : (sft == 1 ? D[0] : kInf);
            if (sft > 2) {                                 // only without the 2:1 guard
                dm1 = kInf;
#pragma unroll
                for (int k = 2; k < W; ++k) if (k == sft - 1) dm1 = D[k];
            }
            if (sft >= 1) {
#pragma unroll
                for (int k = 0; k < W - 1; ++k) D[k] = D[k + 1];
                D[W - 1] = kInf;
            }
            if (sft >= 2) {
#pragma unroll
                for (int k = 0; k < W - 1; ++k) D[k] = D[k + 1];
                D[W - 1] = kInf;
            }
            for (int s = 2; s < min(sft, W); ++s) {        // only without the 2:1 guard
#pragma unroll
                for (int k = 0; k < W - 1; ++k) D[k] = D[k + 1];
                D[W - 1] = kInf;
            }
            PRow a;
            load_row(a, urow, kNrm119, i);
            s32 left = kInf;
#pragma unroll
            for (int k = 0; k < W; ++k) {
                const int j = c - R + k;
                const bool valid = j >= 0 && j < M;
                const s32 up = D[k];
                s32 bst = min(min(up, dm1), left);
                if (i == 0 && j == 0) bst = 0;
                PRow b;
                load_row(b, trow, kNrm119, valid ? j : 0);
                const s32 d = (s32)pdist(a, b);
                const s32 x = (valid && bst < kInf / 2) ? bst + d : kInf;
                dm1 = up;                                  // becomes the diagonal source of cell k+1
                D[k] = x;
                left = x;
            }
            cprev = c;
            err += M;                                      // advance c to floor((i+1)*M/I)
            if (err >= I) { err -= I; ++c; }
            if (err >= I) { err -= I; ++c; }
            if (err >= I) { c += err / I; err %= I; }      // only without the 2:1 guard (M > 2I)
        }
        const int kend = (M - 1) - (cprev - R);            // cell holding column M-1 in the last row
        s32 fin = kInf;
#pragma unroll
        for (int k = 0; k < W; ++k) if (k == kend) fin = D[k];
        return fin < kInf / 2 ? (u32)fin / (u32)(I + M) : SR_DIS_ERR;
    });
}

// ---- K3s: the symmetric slope-constrained DP of Sakoe & Chiba (1978), P = 1 (EXTENSION, parity unpinned) -------------
// g(0,0) = 2 d(0,0); g(i,j) = min(g(i-1,j-2) + 2 d(i,j-1) + d(i,j), g(i-1,j-1) + 2 d(i,j), g(i-2,j-1) + 2 d(i-1,j) + d(i,j))
// over the band of dtw_wide_kernel. A move counts only when its start cell is reachable and the cells it passes through
// (the intermediate cell of a two-step move, and its end) lie in the band; every complete path then weighs I + M, so
// g(I-1, M-1) / (I + M) is a weighted mean of get_dis. Checked against tests/oracle_sym.c.
// One WARP per pair, a whole ROW across the warp, lane l holding columns 4l .. 4l+3 as in dtw_wide_kernel. Row i reads
// only rows i-1 and i-2 of g and row i-1 of d, so there is no in-row recurrence and no scan: a lane needs from the lane
// before it g(i-1, 4l-1) and g(i-1, 4l-2) + 2 d(i, 4l-1) (two shuffles), and g(i-2, 4l-1) is the first of those from the
// previous row. Cells outside the band, or past M, hold d = kSymInf; g is kept clamped to kSymInf. Every move sums at
// most four terms of at most kSymInf = 2^26 (< 2^31), and a reachable g(i,j) <= (i + j + 2) * 65 536 <= 238 * 65 536 <
// 2^24 < kSymInf, so a move is finite exactly when it is below kSymInf.
constexpr s32 kSymInf = 1 << 26;

template <bool kLift>
__global__ void __launch_bounds__(kDtwWarps * 32, 1)       // one CTA per SM (shared memory): up to 128 registers
dtw_sym_kernel(const __grid_constant__ ScanArgs a, const unsigned char *__restrict__ in_ftr, const unsigned char *__restrict__ bank,
               const u8 *__restrict__ status, const u32 *__restrict__ B_dev, const u32 *__restrict__ perm,
               u32 *__restrict__ score, u64 *__restrict__ best) {
    warp_pair_scan<kLift>(a, in_ftr, bank, status, B_dev, perm, score, best, true,
                          [r = a.r](int I, int M, const unsigned char *uslot, const unsigned char *trow, int lane) {
        const int j0 = lane * 4;
        PRow b[4];
        s32 g1[4], g2[4], dp[4];                                       // g(i-1, .), g(i-2, .), d(i-1, .) of the lane's columns
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            load_row(b[k], trow, kNrm119, j0 + k < M ? j0 + k : 0);
            g1[k] = g2[k] = dp[k] = kSymInf;
        }
        s32 w1 = kSymInf;                                              // g(i-2, j0-1): last row's shuffle of g(i-1, j0-1)
        for (int i = 0; i < I; ++i) {
            const int c = (i * M) / I, lo = max(c - r, 0), hi = min(c + r, M - 1);
            PRow a;
            load_row(a, uslot, kNrm119, i);                            // broadcast read
            s32 d[4];
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                const int j = j0 + k;
                d[k] = (j >= lo && j <= hi) ? (s32)pdist(a, b[k]) : kSymInf;
            }
            s32 v1 = __shfl_up_sync(0xFFFFFFFFu, g1[3], 1);                      // g(i-1, j0-1)
            s32 v2 = __shfl_up_sync(0xFFFFFFFFu, g1[2] + 2 * d[3], 1);           // g(i-1, j0-2) + 2 d(i, j0-1)
            if (lane == 0) v1 = v2 = kSymInf;
            const s32 gd[4] = {v1, g1[0], g1[1], g1[2]};                                  // g(i-1, j-1)
            const s32 ga[4] = {v2, v1 + 2 * d[0], g1[0] + 2 * d[1], g1[1] + 2 * d[2]};    // g(i-1, j-2) + 2 d(i, j-1)
            const s32 gc[4] = {w1, g2[0], g2[1], g2[2]};                                  // g(i-2, j-1)
            s32 g[4];
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                s32 x = min(min(ga[k], gc[k] + 2 * dp[k]) + d[k], gd[k] + 2 * d[k]);
                if (i == 0 && j0 + k == 0) x = 2 * d[0];
                g[k] = d[k] < kSymInf ? min(x, kSymInf) : kSymInf;
            }
#pragma unroll
            for (int k = 0; k < 4; ++k) { g2[k] = g1[k]; g1[k] = g[k]; dp[k] = d[k]; }
            w1 = v1;
        }
        const s32 fin = dp_end(g1, (M - 1) & 3, (M - 1) / 4);
        return fin < kSymInf ? (u32)fin / (u32)(I + M) : SR_DIS_ERR;
    });
}

}  // namespace srk

// ---- the one decode of the matcher flags, and the one launcher of the template scan ---------------------------------
bool scan_plan(u32 flags, int band_r, u32 T, bool rules, ScanPlan *out) {
    static_assert(SR_FTR_PER_COMM == 4, "the margin rule's key column is t >> 2");
    // one matcher: the greedy walk, the banded DP with or without SR_DTW_ANY_RATE, or the symmetric DP
    const u32 m = flags & (SR_DTW_BAND | SR_DTW_SYM_P1 | SR_DTW_ANY_RATE);
    if (m != 0 && m != SR_DTW_BAND && m != (SR_DTW_BAND | SR_DTW_ANY_RATE) && m != SR_DTW_SYM_P1) return false;
    const u32 knn = (flags >> 8) & 7u, q = flags >> 16;                // SR_DTW_KNN(k), SR_DTW_REJECT(q)
    if (rules) {
        // sr_set_match's word: of bits 4-15 only the KNN rule's (k <= SR_FTR_PER_COMM) and the lifter; a radius >= 0
        if ((flags & 0xFFF0u & ~SR_DTW_KNN(7) & ~SR_DTW_LIFTER) || knn > SR_FTR_PER_COMM || band_r < 0) return false;
    } else {
        // sr_dtw_batch*: no status to report a rejection in, so no bit >= 16, and bits 4-15 other than the lifter are
        // ignored; a DP's radius must be >= 0 once there are templates to scan
        if (q || (m && T && band_r < 0)) return false;
    }
    ScanPlan &p = *out;
    p.matcher = (m & SR_DTW_SYM_P1) ? ScanPlan::kSym : m ? ScanPlan::kBand : ScanPlan::kGreedy;
    p.tag = (m & SR_DTW_SYM_P1) ? TAG_DTW_SYM : m ? TAG_DTW_BAND : TAG_DTW;
    p.check_sign = flags & SR_DTW_CHECK_SIGN;
    p.guard = !(flags & SR_DTW_ANY_RATE);
    p.lift = flags & SR_DTW_LIFTER;
    // every r >= 118 is the full matrix (|j - c| <= 118 for any two columns), so no r reaches the kernels' c +- r
    p.r = min(band_r, (int)kMaxFrm - 1);
    // under a rule the scan writes a row of C keys per input: one per command for the margin rule alone, one per slot for
    // the KNN rule (ScanArgs); no rule without a status to decide into (rules false) or without a bank
    const u32 C = !rules || !T ? 0 : knn ? T : q ? (T + SR_FTR_PER_COMM - 1) / SR_FTR_PER_COMM : 0;
    p.rule = C ? Rule{C, q, knn} : Rule{0, 0, 0};
    return true;
}

ScanArgs scan_args(const ScanPlan &p, const BankView &bank, const void *in_ftr, u32 B, u32 *score, u64 *best,
                   const u8 *status, const u32 *B_dev) {
    const u32 C = p.rule.C;                                             // the key layout of p.rule (ScanArgs)
    return ScanArgs{static_cast<const unsigned char *>(in_ftr), B, B_dev, status, static_cast<const unsigned char *>(bank.p),
                    bank.n, bank.stride, bank.order, score, best, p.check_sign, p.guard, p.r, C ? C : 1,
                    !C ? 32u : p.rule.knn ? 0u : 2u};
}

#ifndef SR_DTW_VARIANT_DEFAULT
#define SR_DTW_VARIANT_DEFAULT 0
#endif
// the scan under p with the kernels' liftered (kLift) or plain form
template <bool kLift>
static cudaError_t launch_scan_as(sr_handle *h, const ScanPlan &p, const ScanArgs &a) {
    const int num_sms = h->num_sms;
    const cudaStream_t st = h->stream;
    int variant = h->dtw_variant;
    if (variant < 0) {
        static const int env_v = [] { const char *e = getenv("SR_DTW_VARIANT"); return e && *e ? atoi(e) : SR_DTW_VARIANT_DEFAULT; }();
        variant = env_v;
    }
    if (p.matcher == ScanPlan::kGreedy && variant == 1) {
        // dynamic pairs: the longest input (frm_max_kernel, into the handle's scratch word) sizes the ring slots
        cudaError_t e = ensure(h->dtw_scratch, 16);
        if (e != cudaSuccess) return e;
        u32 *max_frm = static_cast<u32 *>(h->dtw_scratch.p);
        e = cudaMemsetAsync(max_frm, 0, 4, st);
        if (e != cudaSuccess) return e;
        const u32 g = min((a.B + 255) / 256, (u32)num_sms * 4u);
        frm_max_kernel<<<g, 256, 0, st>>>(a.in_ftr, a.B, a.status, max_frm, a.B_dev);
        e = cudaGetLastError();
        if (e != cudaSuccess) return e;
        const u32 smem = 226 * 1024;
        e = cudaFuncSetAttribute(dtw_dyn_kernel<kLift>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (e != cudaSuccess) return e;
        return launch_tiles(a.T, [&](u32 tile0, u32 ntiles, int) {
            dtw_dyn_kernel<kLift><<<dim3(ntiles, grid_rows(num_sms, ntiles, a.B, 1u)), kDynWarps * 32, smem, st>>>(
                a, SCAN_PTRS(a), tile0, smem, max_frm);
            return cudaGetLastError();
        });
    }
    if (p.matcher == ScanPlan::kGreedy || (p.matcher == ScanPlan::kBand && p.r == 10)) {
        // lane-packed: one launch per tile width, each with the lane plan of its width
        auto *kernel = p.matcher == ScanPlan::kGreedy ? dtw_kernel<kLift> : dtw_band_thread_kernel<10, kLift>;
        cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 224 * 1024);
        if (e != cudaSuccess) return e;
        return launch_tiles(a.T, [&](u32 tile0, u32 ntiles, int Tt) {
            const LanePlan lp = plan_lanes(Tt);
            kernel<<<dim3(ntiles, grid_rows(num_sms, ntiles, a.B, (u32)(lp.G * lp.NU))), kK2Warps * 32, lp.smem, st>>>(
                a, SCAN_PTRS(a), lp.Wg, lp.NU, lp.G, tile0, Tt);
            return cudaGetLastError();
        });
    }
    // warp per pair: the symmetric DP, the band's warp-scan form for the other r <= 15 (2r+1 lanes of one warp), its
    // whole-row form for r >= 16
    auto *kernel = p.matcher == ScanPlan::kSym ? dtw_sym_kernel<kLift> : p.r <= 15 ? dtw_band_kernel<kLift> : dtw_wide_kernel<kLift>;
    const size_t smem = (size_t)kTileT * kSlotBytes + kTileHdr + (size_t)kDtwWarps * kSlotBytes;
    cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
    const u32 tiles = (a.T + kTileT - 1) / kTileT;
    kernel<<<dim3(tiles, grid_rows(num_sms, tiles, a.B, kDtwWarps)), kDtwWarps * 32, smem, st>>>(a, SCAN_PTRS(a));
    return cudaGetLastError();
}

cudaError_t launch_scan(sr_handle *h, const ScanPlan &p, const ScanArgs &a) {
    if (a.B == 0 || a.T == 0) return cudaSuccess;
    return p.lift ? launch_scan_as<true>(h, p, a) : launch_scan_as<false>(h, p, a);
}
