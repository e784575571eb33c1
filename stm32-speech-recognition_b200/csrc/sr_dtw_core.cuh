// sr_dtw_core.cuh -- the template scan's shared core, used by the static kernels (sr_dtw.cu: greedy dtw_kernel, banded
// dtw_band_kernel, dtw_band_thread_kernel and dtw_wide_kernel, symmetric dtw_sym_kernel) and the dynamic-pair kernel
// (sr_dtw_dyn.cuh): byte-plane rows and their get_dis, the slot header decode, the template tile stager, the greedy walk
// step, the scan's argument block ScanArgs, the score/argmin epilogue, the decision step of the finishers and the launch
// geometry. No kernel here reads the matcher flags: scan_plan (sr_dtw.cu) decodes them once on the host into ScanArgs'
// fields and a Rule, and launch_scan there picks the kernel.
//
// Rows are staged as BYTE PLANES (low bytes | high bytes of the 12 s16), so that
//   sum (a-b)^2 = |a|^2 + |b|^2 - 2 a.b        (exact in Z/2^32, the ring the reference accumulates in)
// costs 12 IDP.4A per local distance on packed registers: a.b = 65536*HH + 256*(HL+LH) + LL.
// A slot holds 24 bytes of planes per row, then one u32 squared norm per row from byte `nrm` on. The static kernels
// size every slot for vv_frm_max rows (nrm = kNrm119); the dynamic kernel sizes them for the longest feature set present.
#pragma once
#include "sr_common.cuh"

namespace srk {

constexpr int kTileT = 32;                                // templates per tile: one CTA column
constexpr u32 kMaxFrm = 119;                              // vv_frm_max
constexpr u32 kNrm119 = kMaxFrm * 24;                     // norm offset of a vv_frm_max-row slot
constexpr int kSlotBytes = kMaxFrm * 24 + 120 * 4;        // rows + squared norms = 3336
constexpr u32 kNoWalk = 0xFFFFFFFFu;                      // frame count of a feature set that is never walked

// ---- byte-plane rows: 6 words = lo bytes of dims 0..11 (3 words) then hi bytes (3 words), plus the squared norm ------
struct PRow { u32 lo[3], hi[3]; u32 n; };

__device__ __forceinline__ void load_row(PRow &r, const unsigned char *slot, u32 nrm, int idx) {
    const uint2 *p = reinterpret_cast<const uint2 *>(slot + idx * 24);
    const uint2 a = p[0], b = p[1], c = p[2];
    r.lo[0] = a.x; r.lo[1] = a.y; r.lo[2] = b.x; r.hi[0] = b.y; r.hi[1] = c.x; r.hi[2] = c.y;
    r.n = reinterpret_cast<const u32 *>(slot + nrm)[idx];
}
__device__ __forceinline__ u32 dp4a_uu(u32 a, u32 b, u32 c) { u32 d; asm("dp4a.u32.u32 %0, %1, %2, %3;" : "=r"(d) : "r"(a), "r"(b), "r"(c)); return d; }
__device__ __forceinline__ u32 dp4a_ss(u32 a, u32 b, u32 c) { u32 d; asm("dp4a.s32.s32 %0, %1, %2, %3;" : "=r"(d) : "r"(a), "r"(b), "r"(c)); return d; }
__device__ __forceinline__ u32 dp4a_su(u32 a, u32 b, u32 c) { u32 d; asm("dp4a.s32.u32 %0, %1, %2, %3;" : "=r"(d) : "r"(a), "r"(b), "r"(c)); return d; }
__device__ __forceinline__ u32 dp4a_us(u32 a, u32 b, u32 c) { u32 d; asm("dp4a.u32.s32 %0, %1, %2, %3;" : "=r"(d) : "r"(a), "r"(b), "r"(c)); return d; }
// get_dis, DTW.C:45-62
__device__ __forceinline__ u32 pdist(const PRow &a, const PRow &b) {
    u32 ll = 0, hh = 0, mx = 0;
#pragma unroll
    for (int j = 0; j < 3; ++j) {
        ll = dp4a_uu(a.lo[j], b.lo[j], ll);
        hh = dp4a_ss(a.hi[j], b.hi[j], hh);
        mx = dp4a_su(a.hi[j], b.lo[j], mx);
        mx = dp4a_us(a.lo[j], b.hi[j], mx);
    }
    const u32 dot = hh * 65536u + mx * 256u + ll;
    return usqrt_trunc(a.n + b.n - 2u * dot);
}
// SR_DTW_LIFTER's transform of one coefficient: sat16(trunc(a * W[c] / 16)), the product in s32
__device__ __forceinline__ u32 lifter16(u32 a, int c) {
    constexpr s32 kW[12] = SR_DTW_LIFTER_W;
    return (u32)min(max(((s32)a * kW[c]) / 16, -32768), 32767);
}
// convert one v_ftr_tag's rows [0,nrows) into the byte-plane slot; threads tid, tid+nthr, ... of the caller. kLift: the
// rows liftered first (SR_DTW_LIFTER), the norms those of the liftered rows
template <bool kLift = false>
__device__ __forceinline__ void stage_planes(unsigned char *slot, u32 nrm, const unsigned char *src_ftr, int nrows, int tid,
                                             int nthr) {
    for (int r = tid; r < nrows; r += nthr) {
        const u32 *s = reinterpret_cast<const u32 *>(src_ftr + 4 + r * 24);
        u32 w[6];
#pragma unroll
        for (int j = 0; j < 6; ++j) w[j] = s[j];
        if constexpr (kLift) {
#pragma unroll
            for (int j = 0; j < 6; ++j) w[j] = pack16(lifter16(lo16s(w[j]), 2 * j), lifter16(hi16s(w[j]), 2 * j + 1));
        }
        u32 lo[3], hi[3], n = 0;
#pragma unroll
        for (int j = 0; j < 3; ++j) {                      // words 2j, 2j+1 hold dims 4j..4j+3
            lo[j] = __byte_perm(w[2 * j], w[2 * j + 1], 0x6420);
            hi[j] = __byte_perm(w[2 * j], w[2 * j + 1], 0x7531);
        }
#pragma unroll
        for (int j = 0; j < 6; ++j) {
            const u32 a = lo16s(w[j]), b = hi16s(w[j]);
            n += a * a + b * b;
        }
        u32 *d = reinterpret_cast<u32 *>(slot + r * 24);
        d[0] = lo[0]; d[1] = lo[1]; d[2] = lo[2]; d[3] = hi[0]; d[4] = hi[1]; d[5] = hi[2];
        reinterpret_cast<u32 *>(slot + nrm)[r] = n;
    }
}

// ---- headers ----------------------------------------------------------------------------------------------------
// frame count from a feature set's first word (save_sign | frm_num << 16), or kNoWalk: a bank slot that is unsigned or
// erased under check_sign (SR_DTW_CHECK_SIGN, main.c:283), or a frm_num > vv_frm_max, whose rows would lie past the
// struct. Utterances pass check_sign = false.
__device__ __forceinline__ u32 decode_frm(u32 hdr, bool check_sign) {
    const u32 frm = hdr >> 16;
    const bool unsigned_slot = check_sign && (hdr & 0xFFFFu) != SR_SAVE_MASK;
    return (unsigned_slot || frm > kMaxFrm) ? kNoWalk : frm;
}
// rows to stage: the greedy do-while may touch row frm, and rows 0 and 1 are always read (DTW.C:146-160), also when
// frm_num == 0. The banded DP reads rows [0, frm) only.
__device__ __forceinline__ int staged_rows(u32 frm) { return frm == kNoWalk ? 0 : (int)min(max(frm + 1u, 2u), kMaxFrm); }
// both sides walkable and, with guard, within the 2:1 length ratio (DTW.C:133). Without it (the banded DP under
// SR_DTW_ANY_RATE) both sides must have at least one frame, which the guard implies for all but the 0:0 pair.
__device__ __forceinline__ bool pair_walks(u32 Iraw, u32 Mraw, bool guard) {
    const int I = (int)Iraw, M = (int)Mraw;
    if (Iraw == kNoWalk || Mraw == kNoWalk) return false;
    return guard ? !(I > M * 2 || 2 * I < M) : (I >= 1 && M >= 1);
}

// ---- the scan's arguments: one block for every template-scan kernel ----------------------------------------------------
// B inputs of kFtrBytes at in_ftr (B_dev: a batch size produced on the device, streaming; status: the per-input SR_ST_*
// gate of the recognition calls, or NULL) against the T bank slots of slot_stride bytes at bank (perm: the slots in
// ascending frm_num order, whose templates of a tile then walk alike, or NULL; results stay under the ORIGINAL slot
// number). score [B][T] and best may be NULL. check_sign, guard (the 2:1 length guard: off only under SR_DTW_ANY_RATE)
// and r (the band radius, at most 118) are the plan's (scan_plan, sr_dtw.cu).
// The argmin key of a pair is (result, bank slot t): strict '<', first wins == lexicographic min. The key of pair (u, t)
// is best[u * key_stride + (t >> key_shift)], the layout the plan's Rule sized:
//   no rule:             one key per input,             key_stride 1,             key_shift 32 (t >> 32 is 0);
//   SR_DTW_REJECT(q):    [B][ceil(T / 4)] per command,  key_stride ceil(T / 4),   key_shift 2. The runner-up command
//                        depends on the winner; the row's minimum is the same argmin key, its second smallest the
//                        runner-up command's score;
//   SR_DTW_KNN(k):       [B][T] per slot, each written once: key_stride T, key_shift 0. A command's score needs all of
//                        its templates' scores.
// Every key starts at (SR_DIS_MAX, slot 0) (main.c:276-278).
// Every scan kernel also takes a's seven pointers as __restrict__ parameters (SCAN_PTRS), which its body reads and
// writes through: only restrict KERNEL parameters keep the loads read-only (LDG.CONSTANT). Restrict-qualified members,
// locals or device-function parameters lose it to the scans' 64-bit atomics and named barriers, and __ldg keeps it but
// changes how the staging loops compile (registers, unrolling).
struct ScanArgs {
    const unsigned char *in_ftr;
    u32 B;
    const u32 *B_dev;
    const u8 *status;
    const unsigned char *bank;
    u32 T, slot_stride;
    const u32 *perm;
    u32 *score;
    u64 *best;
    bool check_sign, guard;
    int r;
    u32 key_stride, key_shift;
};

// The pointers of a, in the order of the scan kernels' __restrict__ parameters
#define SCAN_PTRS(a) (a).in_ftr, (a).bank, (a).status, (a).B_dev, (a).perm, (a).score, (a).best

// stage bank templates t0 .. t0+Tt-1 (bank slot perm[t] when a bank order is given) into tile slots of slot_bytes each:
// planes and norms, frame counts to tfrm[], bank slot numbers to tslot[] unless it is NULL. Warp w of nwarps stages
// templates w, w+nwarps, ... (kLift: liftered, as stage_planes)
template <bool kLift>
__device__ __forceinline__ void stage_tile(unsigned char *tile, u32 slot_bytes, u32 nrm, u32 *tfrm, u32 *tslot,
                                           const unsigned char *bank, u32 slot_stride, bool check_sign, const u32 *perm,
                                           u32 t0, int Tt, int warp, int lane, int nwarps) {
    for (int tt = warp; tt < Tt; tt += nwarps) {
        const u32 ts = perm ? perm[t0 + tt] : t0 + (u32)tt;
        const unsigned char *slot = bank + (size_t)ts * slot_stride;
        const u32 frm = decode_frm(*reinterpret_cast<const u32 *>(slot), check_sign);
        stage_planes<kLift>(tile + (size_t)tt * slot_bytes, nrm, slot, staged_rows(frm), lane, 32);
        if (lane == 0) {
            tfrm[tt] = frm;
            if (tslot) tslot[tt] = ts;
        }
    }
}

// ---- the reference's greedy walk (DTW.C:141-191) over a staged utterance and template -----------------------------
// The walk state lives in the caller's locals, passed by reference: i0/i1 are the utterance rows x-1 and x, m0/m1 the
// template rows y-1 and y, (ya0, yb0) and (ya1, yb1) the dtw_limit intervals of columns x and x+1. (Held in a struct
// across dtw_dyn_kernel's claim/poll loop, the same state compiled to 13 more instructions per step, mostly moves.)
// dtw_limit (DTW.C:76-109) as an open y interval per column: ins(x,y) <=> yb(x) < y < ya(x)
__device__ __forceinline__ int walk_ya(int x, int I, int M, int X1) { return x < X1 ? 2 * x + 2 : (x + (4 - I + 2 * M + 1)) >> 1; }
__device__ __forceinline__ int walk_yb(int x, int I, int M, int X2) { return x < X2 ? (x - 2) >> 1 : 2 * x + (M - 2 * I - 4); }

// first point of the walk of a pair that passed pair_walks (DTW.C:141-146)
__device__ __forceinline__ void greedy_start(int I, int M, int &X1, int &X2, PRow &i0, PRow &i1, PRow &m0, PRow &m1, u32 &dis,
                                             u32 &steps, int &x, int &y, int &ya0, int &yb0, int &ya1, int &yb1,
                                             const unsigned char *urow, u32 unrm, const unsigned char *trow, u32 tnrm) {
    X1 = (2 * M - I) / 3; X2 = (4 * I - 2 * M) / 3;                                              // DTW.C:141-142
    load_row(i0, urow, unrm, 0); load_row(m0, trow, tnrm, 0);
    load_row(i1, urow, unrm, 1); load_row(m1, trow, tnrm, 1);
    dis = pdist(i0, m0);                                                                         // DTW.C:146
    x = 1; y = 1; steps = 1;
    ya0 = walk_ya(1, I, M, X1); yb0 = walk_yb(1, I, M, X2); ya1 = walk_ya(2, I, M, X1); yb1 = walk_yb(2, I, M, X2);
}
// one step of DTW.C:150-188; false once the walk has ended, and its score is then dis / (steps & 0xFFFF) (DTW.C:191,
// step is a u16)
__device__ __forceinline__ bool greedy_step(int I, int M, int X1, int X2, PRow &i0, PRow &i1, PRow &m0, PRow &m1, u32 &dis,
                                            u32 &steps, int &x, int &y, int &ya0, int &yb0, int &ya1, int &yb1,
                                            const unsigned char *urow, u32 unrm, const unsigned char *trow, u32 tnrm) {
    const u32 d_up = pdist(m1, i0), d_right = pdist(m0, i1), d_ru = pdist(m1, i1);
    const u32 up = (y + 1 < ya0 && y + 1 > yb0) ? d_up : SR_DIS_ERR;
    const u32 right = (y < ya1 && y > yb1) ? d_right : SR_DIS_ERR;
    const u32 ru = (y + 1 < ya1 && y + 1 > yb1) ? d_ru : SR_DIS_ERR;
    u32 mn = ru;
    if (mn > right) mn = right;
    if (mn > up) mn = up;
    dis += mn;
    const bool mv_x = (mn == ru) || (mn != up);                                                   // diag, else up, else right
    const bool mv_y = (mn == ru) || (mn == up);
    ++steps;
    if (mv_x) { i0 = i1; ++x; ya0 = ya1; yb0 = yb1; ya1 = walk_ya(x + 1, I, M, X1); yb1 = walk_yb(x + 1, I, M, X2); }
    if (mv_y) { m0 = m1; ++y; }
    if (!(x < I && y < M)) return false;
    if (mv_x) load_row(i1, urow, unrm, x);
    if (mv_y) load_row(m1, trow, tnrm, y);
    return true;
}

// ---- the whole-row (min,+) DP column step (dtw_wide_kernel, align_dp, dtw_connected_kernel, dtw_grammar_kernel) ------
// One warp holds a template column of up to 128 cells, lane l the cells j = 4l .. 4l+3 in D[4]; a step turns the column
// of the previous input row (or frame) into this one. Per cell x_j = d_j + min(A_j, x_{j-1}), A_j = min(up, diag): the
// up and diag terms come from the lane's own D (diag of its first cell by one shuffle), so the in-row recurrence maps a
// lane's incoming x to its outgoing one as f(x) = min(x + a, b) (a = the lane's sum of d, b = its outgoing x for an
// incoming +inf). One warp scan composes these maps, f2(f1(x)) = min(x + a1 + a2, min(b1 + a2, b2)), giving every lane
// its incoming x, and a serial fix-up pass over the lane's four cells writes the column.
// cell(k, up, dg, d, A, valid) fills cell k's local distance d, its A (from up = D(i-1, j) and dg = D(i-1, j-1)) and
// its validity; a cell that is not valid is +inf, and its d still enters the lane's a. fix(k, A, x) sees each cell's A and incoming x = D(i, j-1)
// during the fix-up pass, before the cell is written.
// Headroom of the s32 keys of dtw_wide_kernel and align_dp, +inf = 2^30 - 1: a path to cell (i,j) has at most i+j+1
// cells of at most 65 536, so every reachable cell is below 237 * 65 536 = 15 532 032 and a full-matrix optimum at most
// max(I,M) * 65 536; +inf sums (b1 + a2 <= +inf + 119 * 65 536) stay below 2^31 and are cut back to +inf, so a cell is
// reachable exactly when it is below +inf / 2.
// Headroom of the u64 keys D << 10 | (1023 - start) of dtw_connected_kernel and dtw_grammar_kernel, +inf = 2^62: a word's
// path has at most len + M - 1 <= 818 + 118 cells of get_dis <= 65 535, and at most 818 words each add the penalty
// (< 2^32): D < 119 * 818 * 65 536 + 818 * 2^32 < 2^42, so the end key D << 17 | index << 10 | start fits 59 bits and
// D << 10 plus the row sums of one warp scan (< 128 * 2^26) stays below 2^62.
__device__ __forceinline__ s32 dp_min(s32 a, s32 b) { return min(a, b); }
__device__ __forceinline__ u64 dp_min(u64 a, u64 b) { return a < b ? a : b; }

template <class K, K kInfK, class Cell, class Fix>
__device__ __forceinline__ void dp_column(K (&D)[4], int lane, Cell cell, Fix fix) {
    K dg = __shfl_up_sync(0xFFFFFFFFu, D[3], 1);                     // D(i-1, j0-1)
    if (lane == 0) dg = kInfK;
    K d[4], A[4];
    bool valid[4];
    K x = kInfK, sum = 0;                                            // serial pass for an incoming +inf: b and a
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        cell(k, D[k], dg, d[k], A[k], valid[k]);
        dg = D[k];
        x = valid[k] ? dp_min(d[k] + dp_min(A[k], x), kInfK) : kInfK;
        sum += d[k];
    }
    K fa = sum, fb = x;                                              // inclusive composition of the lanes' maps
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const K pa = __shfl_up_sync(0xFFFFFFFFu, fa, o), pb = __shfl_up_sync(0xFFFFFFFFu, fb, o);
        if (lane >= o) { fb = dp_min(dp_min(pb + fa, fb), kInfK); fa += pa; }
    }
    x = __shfl_up_sync(0xFFFFFFFFu, dp_min(kInfK + fa, fb), 1);     // x_{j0-1}: the previous lanes' maps applied to +inf
    if (lane == 0) x = kInfK;
    x = dp_min(x, kInfK);
#pragma unroll
    for (int k = 0; k < 4; ++k) {                                    // serial fix-up with the true incoming x
        fix(k, A[k], x);
        x = valid[k] ? dp_min(d[k] + dp_min(A[k], x), kInfK) : kInfK;
        D[k] = x;
    }
}
// the end cell D(., M-1) of a column, in every lane: cell kend = (M-1) & 3 of lane lend = (M-1) / 4
template <class K>
__device__ __forceinline__ K dp_end(const K (&D)[4], int kend, int lend) {
    K e = D[0];
#pragma unroll
    for (int k = 1; k < 4; ++k) if (k == kend) e = D[k];
    return __shfl_sync(0xFFFFFFFFu, e, lend);
}

// ---- the argmin keys -----------------------------------------------------------------------------------------------
constexpr u64 kKeyStart = (u64)SR_DIS_MAX << 32;
// a scan under a decision rule writes a row of keys per input
__device__ __forceinline__ bool key_rows(const ScanArgs &a) { return a.key_shift < 32; }
__device__ __forceinline__ u64 *key_of(u64 *best, const ScanArgs &a, u32 u, u32 t) {
    return best + (size_t)u * a.key_stride + ((u64)t >> a.key_shift);
}
// score[u][t] and the spch_recg argmin (main.c:276-291) as one 64-bit atomicMin of the pair's key
__device__ __forceinline__ void emit_pair(u32 *score, u64 *best, const ScanArgs &a, u32 u, u32 t, u32 result) {
    if (score) score[(size_t)u * a.T + t] = result;
    if (best) atomicMin(reinterpret_cast<unsigned long long *>(key_of(best, a, u, t)),
                        (unsigned long long)(((u64)result << 32) | (u64)t));
}

// ---- the margin rule (SR_DTW_REJECT) over one utterance's per-command keys ----------------------------------------
// The two smallest keys of a row of C per-command keys: k1 is the argmin key, k2 the runner-up command's best key
// (~0 when there is no other command). A group of g threads (1, or the 32 lanes of a warp) folds a strided part each and
// merges by shuffles; every lane of the group ends with the row's pair.
struct Top2 { u64 k1, k2; };
__device__ __forceinline__ void top2_add(Top2 &a, u64 k) {
    if (k < a.k1) { a.k2 = a.k1; a.k1 = k; }
    else if (k < a.k2) a.k2 = k;
}
// the same over C keys key(c)
template <class Key>
__device__ __forceinline__ Top2 top2_fold(u32 C, int lane, int g, Key key) {
    Top2 a{~0ull, ~0ull};
    for (u32 c = (u32)lane; c < C; c += (u32)g) top2_add(a, key(c));
    if (g == 32) {
#pragma unroll
        for (int o = 16; o; o >>= 1) {
            const u64 b1 = __shfl_xor_sync(0xFFFFFFFFu, a.k1, o), b2 = __shfl_xor_sync(0xFFFFFFFFu, a.k2, o);
            const u64 lo = a.k1 < b1 ? a.k1 : b1, hi = a.k1 < b1 ? b1 : a.k1, m2 = a.k2 < b2 ? a.k2 : b2;
            a.k1 = lo;
            a.k2 = hi < m2 ? hi : m2;
        }
    }
    return a;
}
__device__ __forceinline__ Top2 top2_row(const u64 *row, u32 C, int lane, int g) {
    return top2_fold(C, lane, g, [row](u32 c) { return row[c]; });
}
// reject a decision of score d1 whose runner-up command scores d2 (SR_DIS_ERR: none): 1000 (d2 - d1) < q d1 in u64
__device__ __forceinline__ bool margin_rejects(u32 d1, u32 d2, u32 q) {
    return d2 != SR_DIS_ERR && 1000ull * (u64)(d2 - d1) < (u64)q * (u64)d1;
}
// threads per utterance of the rule's finishers: one for banks of up to 32 commands, a warp for wider ones
__host__ __device__ __forceinline__ int rule_group(u32 C) { return C > 32 ? 32 : 1; }
// commands of a row of C keys: C per-command keys, or under SR_DTW_KNN (knn > 0) C per-slot keys
__host__ __device__ __forceinline__ u32 rule_cmds(u32 C, u32 knn) { return knn ? (C + SR_FTR_PER_COMM - 1) / SR_FTR_PER_COMM : C; }

// ---- the KNN rule (SR_DTW_KNN) over one utterance's per-slot keys [T] -----------------------------------------------
// Command c's key: its score e_c = floor(sum of the m = min(k, n_c) smallest of its n_c scores that are not SR_DIS_ERR
// / m) (sum in u64), then its slot with the smallest score (the lowest on ties); SR_DIS_ERR << 32 | 0 when n_c = 0.
// A mean of scores below SR_DIS_ERR stays below it, so the lexicographic minimum of the command keys is the decision.
__device__ __forceinline__ u64 knn_key(const u64 *row, u32 T, u32 k, u32 c) {
    u32 s[SR_FTR_PER_COMM];
    u32 t_min = 0, s_min = SR_DIS_ERR;
#pragma unroll
    for (u32 j = 0; j < SR_FTR_PER_COMM; ++j) {
        const u32 t = c * SR_FTR_PER_COMM + j;
        s[j] = t < T ? (u32)(row[t] >> 32) : SR_DIS_ERR;
        if (s[j] < s_min) { s_min = s[j]; t_min = t; }
    }
    // ascending (SR_DIS_ERR, the largest u32, last): a 4-input sorting network
    auto cs = [&](int a, int b) { const u32 lo = min(s[a], s[b]), hi = max(s[a], s[b]); s[a] = lo; s[b] = hi; };
    cs(0, 1); cs(2, 3); cs(0, 2); cs(1, 3); cs(1, 2);
    u32 m = 0;
    u64 sum = 0;
#pragma unroll
    for (u32 j = 0; j < SR_FTR_PER_COMM; ++j)
        if (j < k && s[j] != SR_DIS_ERR) { sum += s[j]; ++m; }
    return m ? ((sum / m) << 32) | t_min : (u64)SR_DIS_ERR << 32;
}
// The decision row of a rule: knn = 0, the margin rule's C per-command keys (top2_row); else the KNN rule's C = T
// per-slot keys, folded per command. k1 is the decision's key (score << 32 | slot), k2 >> 32 the runner-up command's score.
__device__ __forceinline__ Top2 rule_row(const u64 *row, u32 C, u32 knn, int lane, int g) {
    if (!knn) return top2_row(row, C, lane, g);
    return top2_fold(rule_cmds(C, knn), lane, g, [=](u32 c) { return knn_key(row, C, knn, c); });
}

// ---- one record's decision: the step of every finisher (main.c:261-294) -------------------------------------------
// The decision rule of a recognition call, from its matcher flags (scan_plan, sr_dtw.cu): C keys per record (0: no rule,
// one argmin key; else the scan's row, ScanArgs), the margin q of SR_DTW_REJECT(q) and the k of SR_DTW_KNN(k) (0: off).
struct Rule { u32 C, q, knn; };
// threads per record of a finisher: one without a rule (C = 0), else rule_group of the row's commands
__host__ __device__ __forceinline__ u32 rule_lanes(const Rule &rl) { return rl.C ? (u32)rule_group(rule_cmds(rl.C, rl.knn)) : 1u; }
// a finisher's grid of 256-thread CTAs over n records
inline u32 rule_grid(u64 n, const Rule &rl) { return (u32)((n * rule_lanes(rl) + 255) / 256); }
// Record i's decision from its keys and the status st it comes in with. Without a rule (kRule false) its key is keys[i];
// under one the g lanes of its group fold its row of C keys (rule_row), and only lane 0 gets the decision (the others
// return false). An SR_ST_OK decision the margin rule q turns down gets SR_ST_REJECT, and a record whose st is not
// SR_ST_OK reports idx 0 and SR_DIS_ERR.
struct Decision { u64 key; u32 idx, dis, cmd, status; };
template <bool kRule>
__device__ __forceinline__ bool decide(const u64 *keys, u32 i, u32 st, const Rule &rl, u32 g, Decision &d) {
    d.status = st;
    if constexpr (kRule) {
        const u32 lane = threadIdx.x & (g - 1);
        const Top2 t2 = rule_row(keys + (size_t)i * rl.C, rl.C, rl.knn, (int)lane, (int)g);
        if (lane) return false;
        d.key = t2.k1;
        if (st == SR_ST_OK && margin_rejects((u32)(d.key >> 32), (u32)(t2.k2 >> 32), rl.q)) d.status = SR_ST_REJECT;
    } else {
        d.key = keys[i];
    }
    d.idx = (u32)(d.key & 0xFFFFFFFFull);
    d.dis = (u32)(d.key >> 32);
    if (st != SR_ST_OK) { d.idx = 0; d.dis = SR_DIS_ERR; }
    d.cmd = d.idx / SR_FTR_PER_COMM;
    return true;
}

// ---- launch geometry --------------------------------------------------------------------------------------------
// CTA rows per tile column: one CTA per SM over all columns (never a second partial wave), no more than the batch needs
inline u32 grid_rows(int num_sms, u32 ntiles, u32 B, u32 utt_per_cta) {
    u32 gy = (u32)num_sms / ntiles;
    const u32 need = (B + utt_per_cta - 1) / utt_per_cta;
    if (gy > need) gy = need;
    if (gy < 1) gy = 1;
    if (gy > 65535) gy = 65535;
    return gy;
}
// T templates as one launch of the full kTileT-wide tiles and one of the remainder tile: launch(tile0, ntiles, Tt)
template <class Launch>
inline cudaError_t launch_tiles(u32 T, Launch launch) {
    const u32 full = T / kTileT, rem = T % kTileT;
    if (full) {
        cudaError_t e = launch(0u, full, kTileT);
        if (e != cudaSuccess) return e;
    }
    if (rem) return launch(full, 1u, (int)rem);
    return cudaSuccess;
}

}  // namespace srk
