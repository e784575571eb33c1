// sr_long_stream.cu -- K14: live streams of any length (include/sr_long_stream.h). S microphones are fed in chunks for as
// long as they run; every push advances, per stream, exactly what the long-form VAD (sr_vad_long.cu, K11/K12) computes on
// the stream's prefix, and every segment that closes is decided at once, as sr_recognise_long_batch decides it.
//
// One WARP per stream, built from the shared cores (sr_vad_core.cuh):
//   * the chunk is appended to the stream's ring of R samples; a sample that lands in the ring's first M slots is also
//     written to the mirror behind the ring, so every segment that can still be decoded is contiguous in the row;
//   * noise_atap runs once the calibration window is complete (noise_atap_warp);
//   * the new frames are evaluated in windows of at most W frames: the window's blocks are summarised into a per-stream
//     scratch (block_pass over ring slots; one block is summarised again by the next window), then vad_window runs
//     frames_pass over them with last_sig (`cin`) and continues the endpoint FSM from its carried state (open or closed,
//     the run at the edge), both kept in device state (StreamVad, as K4 keeps them) -- K12's loop, cut at push
//     boundaries instead of every 1 024 frames;
//   * a closed segment goes to the push's event list (StreamEvents, shared with K4): its ring offsets, or SR_SEG_NULL
//     when it has more than 119 frames (get_mfcc then gives frm_num 0 and SR_ST_MFCC_FAIL, as the batch call does).
// Recognition is K4's: get_mfcc on the event list with its row map, the status kernel, the handle's matcher and the
// finish kernel, then one D2H copy and one synchronisation (stream_core_recognise, sr_stream.cu).
//
// A pool at a rate other than 8 kHz (sr_long_streams_create_at_rate, include/sr_synth.h) runs one more kernel before the
// step kernel: the resample stage K4 shares (ResampleStage, sr_stream.cu) turns each stream's chunk into the 8 kHz
// outputs whose filter support has arrived, n8(n_in) = resample_ready(n_in) of them in all, with K15's phases and
// arithmetic (sr_resample_core.cuh). The stream's last K - 1 input samples are carried across pushes, so those outputs
// are the first n8 of sr_resample_adc12_dev on everything pushed so far. The step kernel then takes them through its
// ragged path, unchanged.
#include "sr_internal.h"
#include "../../include/sr_long_stream.h"
#include "../../include/sr_synth.h"
#include "sr_vad_core.cuh"

namespace srk {

struct LongStreamState {        // one per stream, device resident
    atap_tag atap;
    u32 n;                      // samples received since the last reset
    u32 calibrated;
    StreamVad vad;
};

// rs_n / rs_hist: the pool's resample stage (at a rate, else NULL), restarted with the stream
__global__ void long_stream_reset_kernel(LongStreamState *st, u32 S, const u8 *which, const atap_tag *atap, u32 *rs_n,
                                         int16_t *rs_hist, u32 hist_stride) {
    const u32 s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= S || (which && !which[s])) return;
    LongStreamState z;
    memset(&z, 0, sizeof z);
    if (atap) z.atap = atap[s];
    z.vad.open_start = SR_SEG_NULL;
    st[s] = z;
    resample_stage_restart(s, rs_n, rs_hist, hist_stride);
}

__global__ void long_stream_query_kernel(const LongStreamState *st, u32 S, u32 *out /* [4][S] */, atap_tag *atap) {
    const u32 s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= S) return;
    const LongStreamState v = st[s];
    out[s] = v.n;
    out[S + s] = v.vad.f.n;
    out[2 * S + s] = v.vad.f.open ? v.vad.open_start : SR_SEG_NULL;
    atap[s] = v.atap;
}

// the FSM's actions on a live stream: remember where the open segment starts; list a closed one as an event
struct StreamCloseAct {
    u32 s, R, frame_len, open_start;
    atap_tag at;
    StreamEvents q;
    __device__ __forceinline__ void open(int, u32, u32 frame) { open_start = 80u * frame; }          // VAD.C:178
    __device__ __forceinline__ void close(int lane, u32 n, u32 frame) {
        if (lane == 0) {
            const u32 st = open_start, end = 80u * frame + 80u, len = end - st;                   // VAD.C:201
            const u32 F = len < frame_len ? 0u : (len - frame_len) / SR_FRAME_MOV + 1u;           // MFCC.C:102-107
            u32 ms = SR_SEG_NULL, me = SR_SEG_NULL;
            if (F >= 1u && F <= SR_VV_FRM_MAX) {
                // ring offset; a start on ring slot 0 is read from the mirror (slot R) so that x[-1] is the real sample in
                // slot R - 1 -- get_mfcc pins x[-1] to mid_val only at row offset 0, which stays stream sample 0
                ms = st % R;
                if (ms == 0 && st != 0) ms = R;
                me = ms + len;
            }
            q.emit(s, n, st, end, ms, me, at);
        }
        open_start = SR_SEG_NULL;
    }
};

constexpr int kLsWarps = 8;

// lens == NULL: every stream receives uniform_len samples; else stream s receives lens[s] (0 = nothing this time).
// Rows of `row` = R + M samples: ring slots [0, R), mirror of slots [0, M) at [R, R + M). info: [S][info_stride] words,
// the summaries of one window's blocks; windows hold at most W frames.
__global__ void __launch_bounds__(kLsWarps * 32, 1)
long_stream_step_kernel(u16 *__restrict__ pcm, u32 R, u32 M, u32 row, u32 S, const u16 *__restrict__ chunk, u32 chunk_stride,
                        u32 uniform_len, const u32 *__restrict__ lens, u32 n_len, LongStreamState *__restrict__ state,
                        u32 *__restrict__ info_all, u32 info_stride, u32 W, u32 frame_len, StreamEventDev *__restrict__ ev,
                        u32 *__restrict__ seg_ev, atap_tag *__restrict__ atap_ev, u32 *__restrict__ map_ev,
                        u32 *__restrict__ n_ev, u32 cap) {
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const u32 s = blockIdx.x * kLsWarps + warp;
    if (s >= S) return;
    LongStreamState *sp = state + s;
    u16 *x = pcm + (size_t)s * row;
    u32 *info = info_all + (size_t)s * info_stride;

    // ---- append the chunk to the ring (len <= max_chunk < R: at most one wrap), then the mirrored slots ---------------
    const u32 n0 = sp->n;
    const u32 len = lens ? lens[s] : uniform_len;
    if (len) {
        const u16 *src = chunk + (size_t)s * chunk_stride;
        const u32 i0 = n0 % R, a = min(len, R - i0);
        warp_copy(x + i0, src, a, lane);
        if (a < len) warp_copy(x, src + a, len - a, lane);
        __syncwarp();
        if (i0 < M) warp_copy(x + R + i0, x + i0, min(a, M - i0), lane);
        if (a < len) warp_copy(x + R, x, min(len - a, M), lane);
        __syncwarp();
    }
    const u32 n = n0 + len;

    // ---- noise_atap as soon as the calibration window is complete (VAD.C:22-71); R >= n_len + max_chunk, so the first
    // n_len samples are still unwrapped in the ring when they complete ------------------------------------------------
    atap_tag at = sp->atap;
    u32 calibrated = sp->calibrated;
    if (!calibrated) {
        if (n_len != 0 && n_len % 240u == 0) {                        // else atap stays as given (VAD.C:33-36)
            if (n < n_len) { if (lane == 0) sp->n = n; return; }
            noise_atap_warp(x, true, n_len, lane, at);
        }
        calibrated = 1;
    }
    const u32 mid = at.mid_val, a_thl = mid + at.n_thl, b_thl = mid - at.n_thl;          // VAD.C:112-113 (u32 wrap)

    // ---- the frames that became complete: frame k once n > 80k + 160 (VAD.C:121), in windows of <= W frames ---------
    const u32 nfr = frames_of(n);
    StreamVad v = sp->vad;
    StreamCloseAct act{s, R, frame_len, v.open_start, at, {ev, seg_ev, map_ev, n_ev, atap_ev, cap}};
    while (v.frames < nfr) {
        const u32 k = v.frames, nw = min(W, nfr - k), nb = nw + 1;  // frame j = blocks j, j + 1
        // block k + i at its ring slot: R is a multiple of 80, so no block straddles the wrap; rows and blocks are 16-byte
        // aligned. The last pass's blocks may run eight lanes per block when they do not wrap.
        auto blk = [&](u32 i) { return x + (u32)((80ull * (k + i)) % R); };
        const u32 last = (nb - 1u) & ~31u;
        block_pass(blk, nb, blk(last) + 80u * (nb - last) <= x + R, true, mid, a_thl, b_thl, info, lane);
        __syncwarp();
        vad_window(info, k, k, nw, lane, at, v.cin, v.f, act);
        __syncwarp();                                                 // the next window rewrites info
        v.frames += nw;
    }
    v.open_start = act.open_start;
    if (lane == 0) {
        sp->atap = at; sp->n = n; sp->calibrated = calibrated;
        sp->vad = v;
    }
}

}  // namespace srk

struct sr_long_stream_pool : StreamCore {
    u32 max_chunk = 0, n_len = 0, R = 0, row = 0, W = 0, info_stride = 0;
    DevBuf pcm, state, info, which, atap0, query;
    std::vector<uint64_t> n_host;                  // samples per stream since its reset, for the 2^32 - 1 limit
    ResampleStage rs;                              // at a rate other than 8 kHz
};

static int long_streams_push_impl(sr_long_stream_pool *p, const uint16_t *chunk, uint32_t chunk_stride, uint32_t uniform_len,
                                  const uint32_t *lens, sr_stream_event *events, uint32_t max_events, uint32_t *n_events) {
    SR_REQUIRE(nullptr, p && n_events);
    sr_handle *h = p->h;
    *n_events = 0;
    const u32 max_len = stream_core_lens(*p, lens, uniform_len);
    SR_REQUIRE(h, max_len == 0 || chunk != nullptr);
    SR_REQUIRE(h, max_len <= p->max_chunk && chunk_stride >= max_len);
    for (u32 s = 0; s < p->S; ++s)                                    // no stream past 2^32 - 1 samples; nothing changes
        if (p->n_host[s] + (lens ? lens[s] : uniform_len) > 0xFFFFFFFFull)
            return fail(h, "sr_long_streams_push: a stream would pass 2^32 - 1 samples", cudaSuccess);
    DeviceGuard g(h->device);
    const u16 *chunk_dev;
    u32 chunk_dev_stride;
    if (const int rc = stream_core_stage(*p, chunk, chunk_stride, max_len, lens != nullptr, &chunk_dev, &chunk_dev_stride)) return rc;
    const u32 *step_lens = (lens && max_len) ? static_cast<const u32 *>(p->lens.p) : nullptr;
    u32 step_uniform = max_len ? uniform_len : 0u;
    if (const int rc = resample_stage_push(p->rs, h, p->S, 0xFFFFFFFFu, &chunk_dev, &chunk_dev_stride, &step_lens, &step_uniform))
        return rc;                                    // at a rate: the step kernel takes the 8 kHz outputs instead
    if (const int rc = launch_on(h, TAG_NONE, "long_stream_step_kernel", [&] {
            long_stream_step_kernel<<<(p->S + kLsWarps - 1) / kLsWarps, kLsWarps * 32, 0, h->stream>>>(
                static_cast<u16 *>(p->pcm.p), p->R, SR_LONG_STREAM_MIRROR, p->row, p->S, chunk_dev, chunk_dev_stride,
                step_uniform, step_lens, p->n_len,
                static_cast<LongStreamState *>(p->state.p), static_cast<u32 *>(p->info.p), p->info_stride, p->W, frame_len(h),
                static_cast<StreamEventDev *>(p->ev.p), static_cast<u32 *>(p->seg_ev.p), static_cast<atap_tag *>(p->atap_ev.p),
                static_cast<u32 *>(p->map_ev.p), static_cast<u32 *>(p->n_ev.p), p->cap);
            return cudaGetLastError();
        }))
        return rc;
    if (max_len)
        for (u32 s = 0; s < p->S; ++s) p->n_host[s] += lens ? lens[s] : uniform_len;
    return stream_core_recognise(*p, static_cast<const u16 *>(p->pcm.p), p->row, events, max_events, n_events);
}

extern "C" {

int sr_long_streams_destroy(sr_long_stream_pool *p) {
    if (!p) return 0;
    DeviceGuard g(p->h->device);
    cudaStreamSynchronize(p->h->stream);
    delete p;                                      // frees its buffers, under g
    return 0;
}

int sr_long_streams_reset(sr_long_stream_pool *p, const uint8_t *which, const atap_tag *atap) {
    SR_REQUIRE(nullptr, p != nullptr);
    sr_handle *h = p->h;
    DeviceGuard g(h->device);
    if (which) SR_CK(h, cudaMemcpyAsync(p->which.p, which, p->S, cudaMemcpyHostToDevice, h->stream));
    if (atap) SR_CK(h, cudaMemcpyAsync(p->atap0.p, atap, (size_t)p->S * sizeof(atap_tag), cudaMemcpyHostToDevice, h->stream));
    if (const int rc = launch_on(h, TAG_NONE, "long_stream_reset_kernel", [&] {
            long_stream_reset_kernel<<<(p->S + 127) / 128, 128, 0, h->stream>>>(
                static_cast<LongStreamState *>(p->state.p), p->S, which ? static_cast<const u8 *>(p->which.p) : nullptr,
                atap ? static_cast<const atap_tag *>(p->atap0.p) : nullptr, static_cast<u32 *>(p->rs.n.p),
                static_cast<int16_t *>(p->rs.hist.p), p->rs.hist_stride);
            return cudaGetLastError();
        }))
        return rc;
    SR_CK(h, cudaStreamSynchronize(h->stream));    // the caller's arrays may go once this returns
    for (u32 s = 0; s < p->S; ++s)
        if (!which || which[s]) p->n_host[s] = 0;
    // events of a restarted stream that are still queued belong to what it was before: they go with it
    std::deque<sr_stream_event> keep;
    for (const sr_stream_event &e : p->pending)
        if (which && !which[e.stream]) keep.push_back(e);
    p->pending.swap(keep);
    return 0;
}

int sr_long_streams_create(sr_handle *h, uint32_t n_streams, uint32_t max_chunk, uint32_t n_len, const atap_tag *atap,
                           sr_long_stream_pool **out) {
    return sr_long_streams_create_at_rate(h, n_streams, max_chunk, n_len, atap, 8000, out);
}

int sr_long_streams_create_at_rate(sr_handle *h, uint32_t n_streams, uint32_t max_chunk, uint32_t n_len, const atap_tag *atap,
                                   uint32_t rate, sr_long_stream_pool **out) {
    SR_REQUIRE(h, h && out && n_streams > 0 && max_chunk >= 1 && max_chunk <= SR_LONG_STREAM_CHUNK_MAX && n_len <= 65535u);
    ResampleRate g;
    SR_REQUIRE(h, resample_rate(rate, &g));
    // max8 = ceil(max_chunk L / M) bounds the 8 kHz samples one push completes: n8(a + b) - n8(a) <= ceil(b L / M)
    const u32 max8 = (u32)(((uint64_t)max_chunk * g.L + g.M - 1) / g.M);
    // events per stream per push: two closings are >= 19 frames apart, a push evaluates at most F new frames
    const u32 c = (n_len != 0 && n_len % 240u == 0) ? n_len : 0u;
    const u32 F = (max8 + c + SR_FRAME_MOV - 1) / SR_FRAME_MOV, E = (F + 18) / 19;
    SR_REQUIRE(h, (uint64_t)n_streams * E < (1ull << 31));
    DeviceGuard g_dev(h->device);
    sr_long_stream_pool *p = new (std::nothrow) sr_long_stream_pool;
    SR_REQUIRE(h, p != nullptr);
    p->max_chunk = max_chunk; p->n_len = n_len;
    const u32 hist = n_len > SR_LONG_STREAM_HISTORY ? n_len : SR_LONG_STREAM_HISTORY;
    p->R = (hist + max8 + 79u) / 80u * 80u;
    p->row = p->R + SR_LONG_STREAM_MIRROR;                            // a multiple of 8: rows start 16-byte aligned
    p->W = std::min(1024u, (max8 + SR_FRAME_MOV - 1) / SR_FRAME_MOV);
    p->info_stride = 2 * (p->W + 1);
    cudaError_t e = cudaSuccess;
    try { p->n_host.assign(n_streams, 0); } catch (...) { e = cudaErrorMemoryAllocation; }
    if (e == cudaSuccess) e = stream_core_alloc(*p, h, n_streams, n_streams * E);
    auto need = [&](DevBuf &b, size_t bytes) { if (e == cudaSuccess) e = ensure(b, bytes); };
    need(p->pcm, (size_t)n_streams * p->row * 2 + 64);
    need(p->state, (size_t)n_streams * sizeof(LongStreamState));
    need(p->info, (size_t)n_streams * p->info_stride * 4);
    need(p->which, n_streams);
    need(p->atap0, (size_t)n_streams * sizeof(atap_tag));
    need(p->query, (size_t)n_streams * (12 + sizeof(atap_tag)));
    if (e == cudaSuccess) e = resample_stage_alloc(p->rs, h, n_streams, rate, max_chunk);
    if (e == cudaSuccess) e = cudaMemsetAsync(p->pcm.p, 0, (size_t)n_streams * p->row * 2 + 64, h->stream);
    if (e != cudaSuccess) { p->h = h; sr_long_streams_destroy(p); return fail(h, "sr_long_streams_create: allocation", e); }
    *out = p;
    return sr_long_streams_reset(p, nullptr, atap);
}

int sr_long_streams_push(sr_long_stream_pool *p, const uint16_t *chunk, uint32_t chunk_len, uint32_t chunk_stride,
                         sr_stream_event *events, uint32_t max_events, uint32_t *n_events) {
    return long_streams_push_impl(p, chunk, chunk_stride, chunk_len, nullptr, events, max_events, n_events);
}

int sr_long_streams_push_ragged(sr_long_stream_pool *p, const uint16_t *chunk, uint32_t chunk_stride, const uint32_t *lens,
                                sr_stream_event *events, uint32_t max_events, uint32_t *n_events) {
    if (!lens) return fail(p ? p->h : nullptr, "sr_long_streams_push_ragged: lens == NULL", cudaSuccess);
    return long_streams_push_impl(p, chunk, chunk_stride, 0, lens, events, max_events, n_events);
}

int sr_long_streams_fetch(sr_long_stream_pool *p, sr_stream_event *events, uint32_t max_events, uint32_t *n_events) {
    SR_REQUIRE(nullptr, p && n_events);
    stream_core_fetch(*p, events, max_events, n_events);
    return 0;
}

uint32_t sr_long_streams_pending(const sr_long_stream_pool *p) { return p ? (uint32_t)p->pending.size() : 0; }
uint32_t sr_long_streams_max_events(const sr_long_stream_pool *p) { return p ? p->cap : 0; }
uint32_t sr_long_streams_ring_len(const sr_long_stream_pool *p) { return p ? p->R : 0; }

int sr_long_streams_state(sr_long_stream_pool *p, uint32_t *n_recv, uint32_t *n_closed, uint32_t *open_start, atap_tag *atap) {
    SR_REQUIRE(nullptr, p != nullptr);
    sr_handle *h = p->h;
    DeviceGuard g(h->device);
    u32 *q = static_cast<u32 *>(p->query.p);
    atap_tag *qa = reinterpret_cast<atap_tag *>(q + 3 * (size_t)p->S);
    if (const int rc = launch_on(h, TAG_NONE, "long_stream_query_kernel", [&] {
            long_stream_query_kernel<<<(p->S + 127) / 128, 128, 0, h->stream>>>(static_cast<const LongStreamState *>(p->state.p),
                                                                               p->S, q, qa);
            return cudaGetLastError();
        }))
        return rc;
    if (n_recv) D2H(h, n_recv, q, (size_t)p->S * 4);
    if (n_closed) D2H(h, n_closed, q + p->S, (size_t)p->S * 4);
    if (open_start) D2H(h, open_start, q + 2 * (size_t)p->S, (size_t)p->S * 4);
    if (atap) D2H(h, atap, qa, (size_t)p->S * sizeof(atap_tag));
    SR_CK(h, cudaStreamSynchronize(h->stream));
    return 0;
}

}  // extern "C"
