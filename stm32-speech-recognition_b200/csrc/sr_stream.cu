// sr_stream.cu -- K4: streaming front end standing in for the reference's blocking capture loop
// (record(), Src/APP/main.c:77-102 + ADC_DMA_Init, Src/BSP/ADC.C:11-103): S concurrent audio streams are fed in
// chunks -- in lock step or each at its own pace -- and every push advances, per stream, exactly the computation the
// reference would do on the finished buffer: noise_atap once the 300 ms calibration window is complete (main.c:258),
// VAD with the reference's carried state (VAD.C:97-218), and every segment the endpoint FSM closes is recognised at
// once (get_mfcc + dtw + argmin, main.c:268-294). After the last chunk the union of the events equals the batch
// result on the complete buffers (segments of sr_vad_batch; segment 0 = sr_recognise_batch). The reference only
// ever recognises segment 0 (main.c:268); here all <= 3 segments are (SURVEY 8f-3).
//
// One WARP per stream, built from the shared VAD steps (sr_vad_core.cuh): the new samples are appended to the stream's
// device row (warp_copy), the 80-sample blocks that became complete are summarised (block_pass) and kept per stream, and
// the frames that became complete are evaluated from them (vad_window), with last_sig and the endpoint FSM's state
// carried from push to push at frame granularity (StreamVad, as K14 carries them). After any push the FSM holds exactly
// the decisions the sequential FSM has taken on the frames seen so far. One push = one H2D copy, five kernels whose batch
// sizes are read from device memory (no host round trip between VAD and recognition), one D2H copy, ONE synchronisation.
//
// A pool at a rate other than 8 kHz (sr_streams_create_at_rate, include/sr_synth.h) runs one more kernel before the step
// kernel: stream_resample_kernel, the resample stage it shares with K14 (ResampleStage, below), turns each stream's chunk
// into the 8 kHz outputs whose filter support has arrived, carrying the stream's last K - 1 inputs across pushes. The
// step kernel takes them through its ragged path, unchanged; outputs past the capture's end are not computed, as the
// step kernel would drop them.
#include "sr_internal.h"
#include "../../include/sr_synth.h"
#include "sr_vad_core.cuh"
#include "sr_dtw_core.cuh"
#include <condition_variable>
#include <deque>

namespace srk {

struct StreamState {            // one per stream, device resident
    atap_tag atap;
    u32 n;                      // samples received
    u32 blocks_done;            // 80-sample blocks summarised
    u32 calibrated;
    u32 seg[6];                 // segments so far, as sr_vad_batch gives them
    StreamVad vad;
};

// rs_n / rs_hist: the pool's resample stage (at a rate, else NULL), restarted with the stream
__global__ void stream_reset_kernel(StreamState *st, u32 S, u32 *rs_n, int16_t *rs_hist, u32 hist_stride) {
    const u32 s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= S) return;
    StreamState z;
    memset(&z, 0, sizeof z);
    for (int i = 0; i < 6; ++i) z.seg[i] = SR_SEG_NULL;
    z.vad.open_start = SR_SEG_NULL;
    st[s] = z;
    resample_stage_restart(s, rs_n, rs_hist, hist_stride);
}

// The FSM's actions on a capture: K0's segments in lanes, and an event for each of the first SR_MAX_VC_CON segments as it
// closes, with the capture's own offsets
struct CaptureAct : SegLanes {
    u32 s, open_start;
    atap_tag at;
    StreamEvents q;
    __device__ __forceinline__ void open(int lane, u32 n, u32 frame) {
        SegLanes::open(lane, n, frame);
        open_start = 80u * frame;
    }
    __device__ __forceinline__ void close(int lane, u32 n, u32 frame) {
        SegLanes::close(lane, n, frame);
        const u32 end = 80u * frame + 80u;
        if (lane == 0 && n < SR_MAX_VC_CON) q.emit(s, n, open_start, end, open_start, end, at);
        open_start = SR_SEG_NULL;
    }
};

constexpr int kStreamWarps = 8;

// lens == NULL: every stream receives uniform_len samples; else stream s receives lens[s] (0 = nothing this time).
// Three CTAs per SM: without that bound ptxas gives the kernel 128 registers (two CTAs); with it 80, no spills.
__global__ void __launch_bounds__(kStreamWarps * 32, 3)
stream_step_kernel(u16 *__restrict__ pcm, u32 L, u32 S, const u16 *__restrict__ chunk, u32 chunk_stride,
                   u32 uniform_len, const u32 *__restrict__ lens, u32 n_len, StreamState *__restrict__ state,
                   u32 *__restrict__ info_all, u32 info_stride, StreamEventDev *__restrict__ ev,
                   u32 *__restrict__ seg_ev /*[cap][2]*/, atap_tag *__restrict__ atap_ev, u32 *__restrict__ map_ev,
                   u32 *__restrict__ n_ev, u32 cap) {
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const u32 s = blockIdx.x * kStreamWarps + warp;
    if (s >= S) return;
    StreamState *sp = state + s;
    u16 *x = pcm + (size_t)s * L;
    u32 *info = info_all + (size_t)s * info_stride;

    // ---- append the new samples to the stream's row ---------------------------------------------------------------
    u32 n = sp->n;
    {
        u32 len = lens ? lens[s] : uniform_len;
        if (len > L - n) len = L - n;                                 // the capture buffer is full (ADC.H:9 VcBuf_Len)
        warp_copy(x + n, chunk + (size_t)s * chunk_stride, len, lane);
        n += len;
        __syncwarp();
    }

    // ---- noise_atap as soon as the calibration window is complete (main.c:258, VAD.C:22-71) -------------------------
    atap_tag at = sp->atap;
    u32 calibrated = sp->calibrated;
    const bool vec_ok = (reinterpret_cast<uintptr_t>(x) & 15) == 0;
    if (!calibrated) {
        if (n < n_len) { if (lane == 0) sp->n = n; return; }
        calibrated = 1;
        if (n_len != 0 && n_len % 240u == 0) noise_atap_warp(x, vec_ok, n_len, lane, at);   // else untouched (VAD.C:33-36)
    }
    const u32 mid = at.mid_val, a_thl = mid + at.n_thl, b_thl = mid - at.n_thl;          // VAD.C:112-113 (u32 wrap)

    // frames i = 80k while i < L-160 (VAD.C:121) over the FINAL buffer length L; frame k = blocks k, k+1
    const u32 nfr_total = frames_of(L);
    const u32 nb_avail = min(n / 80u, nfr_total ? nfr_total + 1 : 0u);

    // ---- summaries of the blocks that became complete (rows and blocks share their alignment: 80 samples = 160 B) ---
    const u32 blocks_done = sp->blocks_done;                           // <= nb_avail: n never decreases
    block_pass([&](u32 i) { return x + 80u * (blocks_done + i); }, nb_avail - blocks_done,
               (reinterpret_cast<uintptr_t>(x) & 3) == 0, vec_ok, mid, a_thl, b_thl, info + 2 * blocks_done, lane);
    __syncwarp();

    // ---- the frames that became complete, the FSM carried from the previous push; events for the segments closed ----
    const u32 ready = nb_avail ? min(nfr_total, nb_avail - 1u) : 0u;
    StreamVad v = sp->vad;
    CaptureAct act{{lane < 6 ? sp->seg[lane] : SR_SEG_NULL}, s, v.open_start, at, {ev, seg_ev, map_ev, n_ev, atap_ev, cap}};
    if (v.frames < ready) {
        vad_window(info, 0u, v.frames, ready - v.frames, lane, at, v.cin, v.f, act);   // <= 818 frames: L <= 65535
        v.frames = ready;
    }
    v.open_start = act.open_start;
    if (lane == 0) {
        sp->atap = at; sp->n = n; sp->blocks_done = nb_avail; sp->calibrated = calibrated;
        sp->vad = v;
    }
    if (lane < 6) sp->seg[lane] = act.seg;
}

__global__ void stream_segments_kernel(const StreamState *st, u32 S, u32 *seg_off, atap_tag *atap, u32 *n_recv) {
    const u32 s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= S) return;
    if (seg_off) for (int i = 0; i < 6; ++i) seg_off[(size_t)s * 6 + i] = st[s].seg[i];
    if (atap) atap[s] = st[s].atap;
    if (n_recv) n_recv[s] = st[s].n;
}

// status per event from the freshly computed features (MFCC fail = frm_num 0, main.c:269-274) + argmin initialiser:
// best[cap] without a decision rule, its C keys per event (ScanArgs) under one (kRule)
template <bool kRule>
__global__ void stream_status_kernel(const unsigned char *ftr, const u32 *n_ev, u32 cap, u8 *status, u32 *frm, u64 *best,
                                     u32 C) {
    const u32 i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= min(*n_ev, cap)) return;
    const u32 f = (*reinterpret_cast<const u32 *>(ftr + (size_t)i * kFtrBytes)) >> 16;
    status[i] = f == 0 ? SR_ST_MFCC_FAIL : SR_ST_OK;
    frm[i] = f;
    if constexpr (kRule) {
        for (u32 c = 0; c < C; ++c) best[(size_t)i * C + c] = kKeyStart;
    } else {
        best[i] = kKeyStart;
    }
}

// each event's decision (decide, under a decision rule when kRule) + one packed record per event for a single D2H copy:
// word 0 of `out` = event count
template <bool kRule>
__global__ void stream_finish_kernel(const StreamEventDev *ev, const u32 *n_ev, u32 cap, const u8 *status, const u32 *frm,
                                     const u64 *best, sr_stream_event *out_rec, u32 *out_count, Rule rl) {
    const u32 g = kRule ? rule_lanes(rl) : 1u;
    const u32 i = (blockIdx.x * blockDim.x + threadIdx.x) / g;
    const u32 ne = min(*n_ev, cap);
    if (i == 0) *out_count = ne;
    if (i >= ne) return;
    Decision d;
    if (!decide<kRule>(best, i, status[i], rl, g, d)) return;
    sr_stream_event r;
    r.stream = ev[i].stream; r.segment = ev[i].segment; r.start = ev[i].start; r.end = ev[i].end;
    r.status = (u8)d.status; r.frm_num = frm[i]; r.best_idx = d.idx; r.best_dis = d.dis; r.cmd = d.cmd;
    out_rec[i] = r;
}

// ---- the resample stage of a pool at a rate: the chunk -> the 8 kHz outputs it completes (K4 and K14) ---------------
constexpr int kRsWarps = 16;
constexpr u32 kRsSpan = 1024;                      // staged input samples per warp and window
constexpr u32 kRsHistMax = 192;                    // K - 1 of the longest phase (48 kHz: 193 taps)
constexpr uint32_t kRates[] = SR_RESAMPLE_RATES;

// outputs per window: T, a multiple of 32, with ceil((T - 1) M / L) + K <= kRsSpan
inline u32 rs_window(const ResampleRate &g) {
    return (u32)(((uint64_t)(kRsSpan - g.K) * g.L / g.M + 1) / 32 * 32);
}

// One warp per stream (a grid-stride loop over streams), lanes over outputs. Stream s has received n0 = rs_n[s] input
// samples and receives len more (lens == NULL: uniform_len); rs_hist holds inputs n0 - H .. n0 - 1 (H = K - 1, centred,
// 0 before sample 0). Outputs [n8(n0), n8(n0 + len)) below index `keep` go to out[s][0, count), count to out_lens[s];
// then the history moves on to the last H inputs. Output k's newest input is j = (kM + c) / L >= n0, its oldest
// j - H >= n0 - H, so history and chunk hold all it reads. The block's shared memory: the rate's [L][K] table, then per
// warp kRsSpan centred inputs of one window of T outputs.
__global__ void __launch_bounds__(kRsWarps * 32)
stream_resample_kernel(const u16 *__restrict__ chunk, u32 chunk_stride, u32 uniform_len, const u32 *__restrict__ lens,
                       u32 S, const int32_t *__restrict__ hp, ResampleRate g, u32 T, u32 keep, u32 *__restrict__ rs_n,
                       int16_t *__restrict__ rs_hist, u32 hist_stride, u16 *__restrict__ out, u32 out_stride,
                       u32 *__restrict__ out_lens) {
    extern __shared__ int32_t rs_smem[];
    int32_t *tab = rs_smem;                                                   // [L][K]
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    int16_t *sx = reinterpret_cast<int16_t *>(rs_smem + g.L * g.K) + warp * kRsSpan;
    for (u32 i = threadIdx.x; i < g.L * g.K; i += blockDim.x) tab[i] = __ldg(hp + i);
    __syncthreads();
    const u32 H = g.K - 1;
    for (u32 s = blockIdx.x * kRsWarps + warp; s < S; s += gridDim.x * kRsWarps) {
        const u32 n0 = rs_n[s], len = lens ? lens[s] : uniform_len;
        const u16 *src = chunk + (size_t)s * chunk_stride;
        int16_t *hist = rs_hist + (size_t)s * hist_stride;
        const uint64_t k0 = min(resample_ready(n0, g.L, g.M, g.c), (uint64_t)keep),
                       k1 = min(resample_ready((uint64_t)n0 + len, g.L, g.M, g.c), (uint64_t)keep);
        u16 *dst = out + (size_t)s * out_stride;
        for (uint64_t kb = k0; kb < k1; kb += T) {
            const u32 nt = (u32)min((uint64_t)T, k1 - kb);
            const uint64_t tb = kb * g.M + g.c;
            const u32 pb = (u32)(tb % g.L);
            const int64_t jb = (int64_t)(tb / g.L), jlo = jb - H;            // newest input of output kb, oldest staged
            const u32 span = (u32)(((uint64_t)(nt - 1) * g.M + pb) / g.L) + g.K;
            for (u32 i = lane; i < span; i += 32) {
                const int64_t d = jlo + i - (int64_t)n0;                      // >= -H
                sx[i] = d < 0 ? hist[d + H] : resample_centre(src[d]);
            }
            __syncwarp();
            for (u32 q = lane; q < nt; q += 32) {
                const u32 u = pb + q * g.M, p = u % g.L;
                const int32_t *h = tab + p * g.K;
                const int16_t *x = sx + H + u / g.L;                           // input jb + u / L
                int32_t acc = 0;
#pragma unroll 4
                for (u32 m = 0; m < g.K; ++m) acc += h[m] * (int32_t)x[-(int32_t)m];
                dst[kb - k0 + q] = resample_code(acc);
            }
            __syncwarp();
        }
        if (lane == 0) { out_lens[s] = (u32)(k1 - k0); rs_n[s] = n0 + len; }
        if (len) {                                                            // inputs n0 + len - H .. n0 + len - 1
            int16_t v[kRsHistMax / 32];
#pragma unroll
            for (u32 t = 0; t < kRsHistMax / 32; ++t) {
                const u32 i = lane + 32 * t;
                const int64_t d = (int64_t)len - H + i;                       // its offset from n0
                v[t] = i >= H ? (int16_t)0 : d < 0 ? hist[d + H] : resample_centre(src[d]);
            }
            __syncwarp();
#pragma unroll
            for (u32 t = 0; t < kRsHistMax / 32; ++t)
                if (lane + 32 * t < H) hist[lane + 32 * t] = v[t];
        }
        __syncwarp();
    }
}

}  // namespace srk

// ---- what every streaming pool shares: the chunk read, recognition of the closed segments, the event queue ----------
cudaError_t stream_core_alloc(StreamCore &c, sr_handle *h, u32 S, u32 cap) {
    c.h = h; c.S = S; c.cap = cap;
    cudaError_t e = cudaSuccess;
    auto need = [&](DevBuf &b, size_t bytes) { if (e == cudaSuccess) e = ensure(b, bytes); };
    need(c.lens, (size_t)S * 4);
    need(c.ev, (size_t)cap * sizeof(StreamEventDev));
    need(c.seg_ev, (size_t)cap * 8);
    need(c.atap_ev, (size_t)cap * sizeof(atap_tag));
    need(c.map_ev, (size_t)cap * 4);
    need(c.n_ev, 16);
    need(c.ftr, (size_t)cap * kFtrBytes);
    need(c.status, cap);
    need(c.frm, (size_t)cap * 4);
    need(c.out, 16 + (size_t)cap * sizeof(sr_stream_event));
    if (e == cudaSuccess) e = c.out_host.alloc(16 + (size_t)cap * sizeof(sr_stream_event));
    if (e == cudaSuccess) e = c.lens_host.alloc((size_t)S * 4);
    return e;
}

u32 stream_core_lens(StreamCore &c, const uint32_t *lens, u32 uniform_len) {
    if (!lens) return uniform_len;
    u32 max_len = 0;
    for (u32 s = 0; s < c.S; ++s) { c.lens_host.p[s] = lens[s]; if (lens[s] > max_len) max_len = lens[s]; }
    return max_len;
}

int stream_core_stage(StreamCore &c, const uint16_t *chunk, u32 chunk_stride, u32 max_len, bool ragged, const u16 **chunk_dev_out,
                      u32 *chunk_dev_stride_out) {
    sr_handle *h = c.h;
    if (h->comm) { const int rc = sr_comm_wait(h); if (rc) return rc; }   // a pending gather may still read the handle's key buffer
    const u16 *chunk_dev = static_cast<const u16 *>(c.stage.p);
    u32 chunk_dev_stride = c.stage_stride;
    if (max_len) {
        // Pinned (cudaHostAlloc / cudaHostRegister / sr_host_alloc*) chunks are read by the kernel straight from host memory:
        // one coalesced 16-byte-per-lane read per stream row, no copy-engine descriptor per row (a strided [S][chunk] slice
        // of a larger capture array is 8192 rows of a few hundred bytes: the 2-D copy alone took ~2 ms). Pageable memory
        // goes through a device staging buffer.
        cudaPointerAttributes attr;
        bool zero_copy = false;
        if (cudaPointerGetAttributes(&attr, chunk) == cudaSuccess && attr.type == cudaMemoryTypeHost && attr.devicePointer) {
            chunk_dev = static_cast<const u16 *>(attr.devicePointer);
            chunk_dev_stride = chunk_stride;
            zero_copy = true;
        } else cudaGetLastError();
        if (!zero_copy) {
            const u32 sstride = (max_len + 7u) & ~7u;                    // staging rows start 16-byte aligned
            SR_CK(h, ensure(c.stage, (size_t)c.S * sstride * 2 + 64));
            c.stage_stride = sstride;
            chunk_dev = static_cast<const u16 *>(c.stage.p); chunk_dev_stride = sstride;
            SR_CK(h, cudaMemcpy2DAsync(c.stage.p, (size_t)sstride * 2, chunk, (size_t)chunk_stride * 2, (size_t)max_len * 2, c.S,
                                       cudaMemcpyHostToDevice, h->stream));
        }
        if (ragged) SR_CK(h, cudaMemcpyAsync(c.lens.p, c.lens_host.p, (size_t)c.S * 4, cudaMemcpyHostToDevice, h->stream));
    }
    SR_CK(h, cudaMemsetAsync(c.n_ev.p, 0, 4, h->stream));
    *chunk_dev_out = chunk_dev;
    *chunk_dev_stride_out = chunk_dev_stride;
    return 0;
}

int stream_core_recognise(StreamCore &c, const u16 *pcm, u32 row_len, sr_stream_event *events, u32 max_events, u32 *n_events) {
    sr_handle *h = c.h;
    u32 *n_ev = static_cast<u32 *>(c.n_ev.p);
    // recognise the closed segments; every kernel reads the number of events from device memory (upper bound: cap)
    SR_LAUNCH(h, TAG_NONE, launch_mfcc_h(h, pcm, row_len, c.cap, static_cast<const u32 *>(c.seg_ev.p), 2,
                                         static_cast<const atap_tag *>(c.atap_ev.p), c.ftr.p, static_cast<const u32 *>(c.map_ev.p),
                                         c.S, n_ev));
    ScanPlan p;                                                          // the handle's matcher, read at every push
    scan_plan(SR_DTW_CHECK_SIGN | h->match_flags, h->match_r, h->bank.n, true, &p);   // flags sr_set_match accepted
    const u32 C = p.rule.C;
    SR_CK(h, ensure(h->best, (size_t)c.cap * (C ? C : 1) * 8));
    u64 *best = static_cast<u64 *>(h->best.p);
    const u32 gb = (c.cap + 255) / 256;
    if (const int rc = launch_on(h, TAG_NONE, "stream_status_kernel", [&] {
            (C ? stream_status_kernel<true> : stream_status_kernel<false>)<<<gb, 256, 0, h->stream>>>(
                static_cast<const unsigned char *>(c.ftr.p), n_ev, c.cap, static_cast<u8 *>(c.status.p),
                static_cast<u32 *>(c.frm.p), best, C);
            return cudaGetLastError();
        }))
        return rc;
    if (h->bank.n)
        SR_LAUNCH(h, TAG_NONE, launch_scan(h, p, scan_args(p, h->bank, c.ftr.p, c.cap, nullptr, best,
                                                           static_cast<const u8 *>(c.status.p), n_ev)));
    u32 *out_count = static_cast<u32 *>(c.out.p);
    sr_stream_event *out_rec = reinterpret_cast<sr_stream_event *>(static_cast<unsigned char *>(c.out.p) + 16);
    if (const int rc = launch_on(h, TAG_NONE, "stream_finish_kernel", [&] {
            (C ? stream_finish_kernel<true> : stream_finish_kernel<false>)<<<rule_grid(c.cap, p.rule), 256, 0, h->stream>>>(
                static_cast<const StreamEventDev *>(c.ev.p), n_ev, c.cap, static_cast<const u8 *>(c.status.p),
                static_cast<const u32 *>(c.frm.p), best, out_rec, out_count, p.rule);
            return cudaGetLastError();
        }))
        return rc;
    const u32 quick = c.cap < StreamCore::kQuick ? c.cap : StreamCore::kQuick;
    D2H(h, c.out_host.p, c.out.p, 16 + (size_t)quick * sizeof(sr_stream_event));
    SR_CK(h, cudaStreamSynchronize(h->stream));                       // the one synchronisation of a push
    const u32 ne = *reinterpret_cast<const u32 *>(c.out_host.p);
    if (ne > quick) {                                                 // rare: a burst of closings larger than the quick window
        D2H(h, c.out_host.p + 16 + (size_t)quick * sizeof(sr_stream_event), static_cast<unsigned char *>(c.out.p) + 16 + (size_t)quick * sizeof(sr_stream_event),
            (size_t)(ne - quick) * sizeof(sr_stream_event));
        SR_CK(h, cudaStreamSynchronize(h->stream));
    }
    const sr_stream_event *rec = reinterpret_cast<const sr_stream_event *>(c.out_host.p + 16);
    u32 k = 0;
    // older queued events first, then this push's; whatever does not fit stays queued for the pool's fetch call
    while (k < max_events && events && !c.pending.empty()) { events[k++] = c.pending.front(); c.pending.pop_front(); }
    u32 i = 0;
    if (c.pending.empty()) for (; i < ne && k < max_events && events; ++i) events[k++] = rec[i];
    for (; i < ne; ++i) c.pending.push_back(rec[i]);
    *n_events = k;
    return 0;
}

void stream_core_fetch(StreamCore &c, sr_stream_event *events, u32 max_events, u32 *n_events) {
    u32 k = 0;
    while (k < max_events && events && !c.pending.empty()) { events[k++] = c.pending.front(); c.pending.pop_front(); }
    *n_events = k;
}

cudaError_t resample_stage_alloc(ResampleStage &r, sr_handle *h, u32 S, u32 rate, u32 max_in) {
    ResampleRate g;
    if (rate == 8000 || !resample_rate(rate, &g)) return cudaSuccess;
    const int32_t *hp = resample_phases(rate, h->device);
    if (!hp) return cudaErrorMemoryAllocation;
    r.rate = g; r.hp = hp;
    r.T = rs_window(g);
    const u32 max8 = (u32)(((uint64_t)max_in * g.L + g.M - 1) / g.M);  // the most 8 kHz samples one push completes
    r.out_stride = (max8 + 7u) & ~7u;                                   // staging rows start 16-byte aligned
    r.hist_stride = (g.K - 1 + 7u) & ~7u;
    r.smem = (size_t)g.L * g.K * 4 + (size_t)kRsWarps * kRsSpan * 2;
    const u32 blocks = (S + kRsWarps - 1) / kRsWarps, per_sm = (u32)(200u * 1024u / r.smem);
    r.grid = std::min(blocks, (u32)h->num_sms * std::max(per_sm, 1u));
    cudaError_t e = cudaSuccess;
    auto need = [&](DevBuf &b, size_t bytes) { if (e == cudaSuccess) e = ensure(b, bytes); };
    need(r.out, (size_t)S * r.out_stride * 2 + 64);
    need(r.lens, (size_t)S * 4);
    need(r.n, (size_t)S * 4);
    need(r.hist, (size_t)S * r.hist_stride * 2);
    // the limit every rate needs, the same value whichever pool sets it: pools at other rates may be launching
    size_t smem_max = 0;
    for (const uint32_t v : kRates) {
        ResampleRate q;
        if (resample_rate(v, &q)) smem_max = std::max(smem_max, (size_t)q.L * q.K * 4 + (size_t)kRsWarps * kRsSpan * 2);
    }
    if (e == cudaSuccess)
        e = cudaFuncSetAttribute(stream_resample_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_max);
    return e;
}

int resample_stage_push(ResampleStage &r, sr_handle *h, u32 S, u32 keep, const u16 **chunk, u32 *stride, const u32 **lens,
                        u32 *uniform_len) {
    if (!r.hp) return 0;
    if (const int rc = launch_on(h, TAG_NONE, "stream_resample_kernel", [&] {
            stream_resample_kernel<<<r.grid, kRsWarps * 32, r.smem, h->stream>>>(
                *chunk, *stride, *uniform_len, *lens, S, r.hp, r.rate, r.T, keep, static_cast<u32 *>(r.n.p),
                static_cast<int16_t *>(r.hist.p), r.hist_stride, static_cast<u16 *>(r.out.p), r.out_stride,
                static_cast<u32 *>(r.lens.p));
            return cudaGetLastError();
        }))
        return rc;
    *chunk = static_cast<const u16 *>(r.out.p);
    *stride = r.out_stride;
    *lens = static_cast<const u32 *>(r.lens.p);
    *uniform_len = 0;
    return 0;
}

struct sr_stream_pool : StreamCore {
    u32 L = 0, n_len = 0, info_stride = 0;
    u32 max_in = 0;                                // the longest chunk in input samples: L at 8 kHz
    DevBuf pcm, state, info;
    ResampleStage rs;                              // at a rate other than 8 kHz
    std::vector<uint64_t> n_in;                    // at a rate: input samples per stream since the reset, for 2^32 - 1
};

static int streams_push_impl(sr_stream_pool *p, const uint16_t *chunk, uint32_t chunk_stride, uint32_t uniform_len,
                             const uint32_t *lens, sr_stream_event *events, uint32_t max_events, uint32_t *n_events);

extern "C" {

int sr_streams_destroy(sr_stream_pool *p) {
    if (!p) return 0;
    DeviceGuard g(p->h->device);
    cudaStreamSynchronize(p->h->stream);
    delete p;                                      // frees its buffers, under g
    return 0;
}

int sr_streams_reset(sr_stream_pool *p) {
    SR_REQUIRE(nullptr, p != nullptr);
    sr_handle *h = p->h;
    DeviceGuard g(h->device);
    p->pending.clear();
    if (const int rc = launch_on(h, TAG_NONE, "stream_reset_kernel", [&] {
            stream_reset_kernel<<<(p->S + 127) / 128, 128, 0, h->stream>>>(static_cast<StreamState *>(p->state.p), p->S,
                                                                          static_cast<u32 *>(p->rs.n.p),
                                                                          static_cast<int16_t *>(p->rs.hist.p), p->rs.hist_stride);
            return cudaGetLastError();
        }))
        return rc;
    std::fill(p->n_in.begin(), p->n_in.end(), 0);
    SR_CK(h, cudaMemsetAsync(p->pcm.p, 0, (size_t)p->S * p->L * 2, h->stream));
    return 0;
}

int sr_streams_create(sr_handle *h, uint32_t n_streams, uint32_t max_samples, uint32_t n_len, sr_stream_pool **out) {
    return sr_streams_create_at_rate(h, n_streams, max_samples, n_len, 8000, out);
}

int sr_streams_create_at_rate(sr_handle *h, uint32_t n_streams, uint32_t max_samples, uint32_t n_len, uint32_t rate,
                              sr_stream_pool **out) {
    SR_REQUIRE(h, h && out && n_streams > 0 && max_samples > 0 && max_samples <= 65535u && n_len <= max_samples);
    ResampleRate rg;
    SR_REQUIRE(h, resample_rate(rate, &rg));
    DeviceGuard g(h->device);
    sr_stream_pool *p = new (std::nothrow) sr_stream_pool;
    SR_REQUIRE(h, p != nullptr);
    p->L = max_samples; p->n_len = n_len;
    // the longest chunk completes at most max_samples 8 kHz samples: n8(a + b) - n8(a) <= ceil(b L / M) <= max_samples
    p->max_in = (u32)(((uint64_t)max_samples * rg.M) / rg.L);
    p->info_stride = 2 * (max_samples / 80 + 2);
    cudaError_t e = stream_core_alloc(*p, h, n_streams, 3 * n_streams);
    auto need = [&](DevBuf &b, size_t bytes) { if (e == cudaSuccess) e = ensure(b, bytes); };
    need(p->pcm, (size_t)n_streams * max_samples * 2 + 64);
    need(p->state, (size_t)n_streams * sizeof(StreamState));
    need(p->info, (size_t)n_streams * p->info_stride * 4);
    if (e == cudaSuccess) e = resample_stage_alloc(p->rs, h, n_streams, rate, p->max_in);
    if (e == cudaSuccess && p->rs.hp) { try { p->n_in.assign(n_streams, 0); } catch (...) { e = cudaErrorMemoryAllocation; } }
    if (e != cudaSuccess) { sr_streams_destroy(p); return fail(h, "sr_streams_create: allocation", e); }
    *out = p;
    return sr_streams_reset(p);
}

// Append chunk_len samples to every stream (chunk[s*chunk_stride + i], host memory; pinned for best latency),
// advance VAD, recognise every segment that closed. Returns after the results are on the host.
int sr_streams_push(sr_stream_pool *p, const uint16_t *chunk, uint32_t chunk_len, uint32_t chunk_stride,
                    sr_stream_event *events, uint32_t max_events, uint32_t *n_events) {
    return streams_push_impl(p, chunk, chunk_stride, chunk_len, nullptr, events, max_events, n_events);
}

// The same with one length per stream: stream s receives lens[s] samples (chunk[s*chunk_stride .. + lens[s])), 0 = none.
int sr_streams_push_ragged(sr_stream_pool *p, const uint16_t *chunk, uint32_t chunk_stride, const uint32_t *lens,
                           sr_stream_event *events, uint32_t max_events, uint32_t *n_events) {
    if (!lens) return fail(p ? p->h : nullptr, "sr_streams_push_ragged: lens == NULL", cudaSuccess);
    return streams_push_impl(p, chunk, chunk_stride, 0, lens, events, max_events, n_events);
}

// events queued by earlier pushes whose caller buffer was too small (nothing is ever dropped)
int sr_streams_fetch(sr_stream_pool *p, sr_stream_event *events, uint32_t max_events, uint32_t *n_events) {
    SR_REQUIRE(nullptr, p && n_events);
    stream_core_fetch(*p, events, max_events, n_events);
    return 0;
}
uint32_t sr_streams_pending(const sr_stream_pool *p) { return p ? (uint32_t)p->pending.size() : 0; }

// segments (and atap, samples received) found so far: same layout as sr_vad_batch's output; host pointers, may be NULL
int sr_streams_segments(sr_stream_pool *p, uint32_t *seg_off, atap_tag *atap) {
    SR_REQUIRE(nullptr, p != nullptr);
    sr_handle *h = p->h;
    DeviceGuard g(h->device);
    SR_CK(h, ensure(h->seg, (size_t)p->S * 24));
    SR_CK(h, ensure(h->atap, (size_t)p->S * sizeof(atap_tag)));
    if (const int rc = launch_on(h, TAG_NONE, "stream_segments_kernel", [&] {
            stream_segments_kernel<<<(p->S + 127) / 128, 128, 0, h->stream>>>(static_cast<const StreamState *>(p->state.p), p->S,
                                                                             static_cast<u32 *>(h->seg.p),
                                                                             static_cast<atap_tag *>(h->atap.p), nullptr);
            return cudaGetLastError();
        }))
        return rc;
    if (seg_off) D2H(h, seg_off, h->seg.p, (size_t)p->S * 24);
    if (atap) D2H(h, atap, h->atap.p, (size_t)p->S * sizeof(atap_tag));
    SR_CK(h, cudaStreamSynchronize(h->stream));
    return 0;
}

}  // extern "C"

static int streams_push_impl(sr_stream_pool *p, const uint16_t *chunk, uint32_t chunk_stride, uint32_t uniform_len,
                             const uint32_t *lens, sr_stream_event *events, uint32_t max_events, uint32_t *n_events) {
    SR_REQUIRE(nullptr, p && n_events);
    sr_handle *h = p->h;
    *n_events = 0;
    const u32 max_len = stream_core_lens(*p, lens, uniform_len);
    SR_REQUIRE(h, max_len == 0 || chunk != nullptr);
    SR_REQUIRE(h, max_len <= p->max_in && chunk_stride >= max_len);
    if (p->rs.hp)                                                     // no input count past 2^32 - 1; nothing changes
        for (u32 s = 0; s < p->S; ++s)
            if (p->n_in[s] + (lens ? lens[s] : uniform_len) > 0xFFFFFFFFull)
                return fail(h, "sr_streams_push: a stream would pass 2^32 - 1 input samples", cudaSuccess);
    DeviceGuard g(h->device);
    const u16 *chunk_dev;
    u32 chunk_dev_stride;
    if (const int rc = stream_core_stage(*p, chunk, chunk_stride, max_len, lens != nullptr, &chunk_dev, &chunk_dev_stride)) return rc;
    const u32 *step_lens = (lens && max_len) ? static_cast<const u32 *>(p->lens.p) : nullptr;
    u32 step_uniform = max_len ? uniform_len : 0u;
    // at a rate: the step kernel takes the 8 kHz outputs instead, none past the capture's end (it would drop them)
    if (const int rc = resample_stage_push(p->rs, h, p->S, p->L, &chunk_dev, &chunk_dev_stride, &step_lens, &step_uniform))
        return rc;
    u32 *n_ev = static_cast<u32 *>(p->n_ev.p);
    if (const int rc = launch_on(h, TAG_NONE, "stream_step_kernel", [&] {
            stream_step_kernel<<<(p->S + kStreamWarps - 1) / kStreamWarps, kStreamWarps * 32, 0, h->stream>>>(
                static_cast<u16 *>(p->pcm.p), p->L, p->S, chunk_dev, chunk_dev_stride, step_uniform, step_lens, p->n_len,
                static_cast<StreamState *>(p->state.p), static_cast<u32 *>(p->info.p), p->info_stride,
                static_cast<StreamEventDev *>(p->ev.p), static_cast<u32 *>(p->seg_ev.p), static_cast<atap_tag *>(p->atap_ev.p),
                static_cast<u32 *>(p->map_ev.p), n_ev, p->cap);
            return cudaGetLastError();
        }))
        return rc;
    if (p->rs.hp && max_len)
        for (u32 s = 0; s < p->S; ++s) p->n_in[s] += lens ? lens[s] : uniform_len;
    return stream_core_recognise(*p, static_cast<const u16 *>(p->pcm.p), p->L, events, max_events, n_events);
}

// ---- streams sharded over several handles / GPUs (BASELINE configs[4] on 8 GPUs) ---------------------------------
// Streams [S*g/G, S*(g+1)/G) live on handles[g]. One persistent host thread per shard issues that shard's push, so
// the G pushes (copies, kernels, the one synchronisation each) run concurrently; events come back with global stream
// indices, shard after shard.
struct sr_stream_group {
    struct Shard {
        sr_stream_pool *pool = nullptr;
        u32 s0 = 0, S = 0;
        std::thread th;
        std::mutex m;
        std::condition_variable cv;
        bool go = false, done = false, stop = false;
        const uint16_t *chunk = nullptr;
        const uint32_t *lens = nullptr;
        u32 stride = 0, ulen = 0;
        std::vector<sr_stream_event> ev;
        u32 ne = 0;
        int rc = 0;
    };
    std::vector<Shard *> shards;
    u32 S = 0;
};

static void group_worker(sr_stream_group::Shard *sh) {
    sr_bind_thread_to_device(sh->pool->h->device);                    // feed the GPU from its own socket
    for (;;) {
        std::unique_lock<std::mutex> lk(sh->m);
        sh->cv.wait(lk, [&] { return sh->go || sh->stop; });
        if (sh->stop) return;
        sh->go = false;
        lk.unlock();
        sh->rc = streams_push_impl(sh->pool, sh->chunk, sh->stride, sh->ulen, sh->lens, sh->ev.data(), (u32)sh->ev.size(), &sh->ne);
        lk.lock();
        sh->done = true;
        sh->cv.notify_all();
    }
}

extern "C" {

int sr_stream_group_destroy(sr_stream_group *gr) {
    if (!gr) return 0;
    for (auto *sh : gr->shards) {
        if (sh->th.joinable()) {
            { std::lock_guard<std::mutex> lk(sh->m); sh->stop = true; }
            sh->cv.notify_all();
            sh->th.join();
        }
        sr_streams_destroy(sh->pool);
        delete sh;
    }
    delete gr;
    return 0;
}

int sr_stream_group_create(sr_handle *const *handles, uint32_t n_handles, uint32_t n_streams, uint32_t max_samples,
                           uint32_t n_len, sr_stream_group **out) {
    return sr_stream_group_create_at_rate(handles, n_handles, n_streams, max_samples, n_len, 8000, out);
}

int sr_stream_group_create_at_rate(sr_handle *const *handles, uint32_t n_handles, uint32_t n_streams, uint32_t max_samples,
                                   uint32_t n_len, uint32_t rate, sr_stream_group **out) {
    ResampleRate rg;
    if (!handles || !out || n_handles == 0 || n_streams < n_handles || !resample_rate(rate, &rg))
        return fail(nullptr, "sr_stream_group_create: bad arguments", cudaSuccess);
    sr_stream_group *gr = new (std::nothrow) sr_stream_group;
    if (!gr) return fail(nullptr, "sr_stream_group_create: out of memory", cudaErrorMemoryAllocation);
    gr->S = n_streams;
    for (u32 g = 0; g < n_handles; ++g) {
        auto *sh = new sr_stream_group::Shard;
        sh->s0 = (u32)((uint64_t)n_streams * g / n_handles);
        sh->S = (u32)((uint64_t)n_streams * (g + 1) / n_handles) - sh->s0;
        gr->shards.push_back(sh);
        const int rc = sr_streams_create_at_rate(handles[g], sh->S, max_samples, n_len, rate, &sh->pool);
        if (rc) { sr_stream_group_destroy(gr); return rc; }
        sh->ev.resize(3 * (size_t)sh->S);
        sh->th = std::thread(group_worker, sh);
    }
    *out = gr;
    return 0;
}

int sr_stream_group_reset(sr_stream_group *gr) {
    if (!gr) return fail(nullptr, "sr_stream_group_reset: NULL", cudaSuccess);
    for (auto *sh : gr->shards) { const int rc = sr_streams_reset(sh->pool); if (rc) return rc; }
    return 0;
}

static int group_push(sr_stream_group *gr, const uint16_t *chunk, uint32_t stride, uint32_t ulen, const uint32_t *lens,
                      sr_stream_event *events, uint32_t max_events, uint32_t *n_events) {
    if (!gr || !n_events) return fail(nullptr, "sr_stream_group_push: bad arguments", cudaSuccess);
    *n_events = 0;
    for (auto *sh : gr->shards)                                       // every shard must recognise with the same matcher
        if (!same_match(sh->pool->h, gr->shards[0]->pool->h))
            return fail(nullptr, "sr_stream_group_push: handles differ in their matcher", cudaSuccess);
    for (auto *sh : gr->shards) {
        std::lock_guard<std::mutex> lk(sh->m);
        sh->chunk = chunk ? chunk + (size_t)sh->s0 * stride : nullptr;
        sh->lens = lens ? lens + sh->s0 : nullptr;
        sh->stride = stride; sh->ulen = ulen; sh->done = false; sh->go = true;
        sh->cv.notify_all();
    }
    u32 k = 0;
    int rc = 0;
    for (auto *sh : gr->shards) {
        std::unique_lock<std::mutex> lk(sh->m);
        sh->cv.wait(lk, [&] { return sh->done; });
        if (sh->rc && !rc) rc = sh->rc;
        for (u32 i = 0; i < sh->ne; ++i) {
            sr_stream_event e = sh->ev[i];
            e.stream += sh->s0;
            if (events && k < max_events) events[k++] = e;
            else { e.stream -= sh->s0; sh->pool->pending.push_back(e); }    // handed out (oldest first) by this shard's next push
        }
    }
    *n_events = k;
    return rc;
}

int sr_stream_group_push(sr_stream_group *gr, const uint16_t *chunk, uint32_t chunk_len, uint32_t chunk_stride,
                         sr_stream_event *events, uint32_t max_events, uint32_t *n_events) {
    return group_push(gr, chunk, chunk_stride, chunk_len, nullptr, events, max_events, n_events);
}
int sr_stream_group_push_ragged(sr_stream_group *gr, const uint16_t *chunk, uint32_t chunk_stride, const uint32_t *lens,
                                sr_stream_event *events, uint32_t max_events, uint32_t *n_events) {
    if (!lens) return fail(nullptr, "sr_stream_group_push_ragged: lens == NULL", cudaSuccess);
    return group_push(gr, chunk, chunk_stride, 0, lens, events, max_events, n_events);
}
int sr_stream_group_segments(sr_stream_group *gr, uint32_t *seg_off, atap_tag *atap) {
    if (!gr) return fail(nullptr, "sr_stream_group_segments: NULL", cudaSuccess);
    for (auto *sh : gr->shards) {
        const int rc = sr_streams_segments(sh->pool, seg_off ? seg_off + (size_t)sh->s0 * 6 : nullptr, atap ? atap + sh->s0 : nullptr);
        if (rc) return rc;
    }
    return 0;
}

}  // extern "C"
