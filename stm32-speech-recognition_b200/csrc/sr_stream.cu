// sr_stream.cu -- K4: streaming front end standing in for the reference's blocking capture loop
// (record(), Src/APP/main.c:77-102 + ADC_DMA_Init, Src/BSP/ADC.C:11-103): S concurrent audio streams are fed in
// chunks -- in lock step or each at its own pace -- and every push advances, per stream, exactly the computation the
// reference would do on the finished buffer: noise_atap once the 300 ms calibration window is complete (main.c:258),
// VAD with the reference's carried state (VAD.C:97-218), and every segment the endpoint FSM closes is recognised at
// once (get_mfcc + dtw + argmin, main.c:268-294). After the last chunk the union of the events equals the batch
// result on the complete buffers (segments of sr_vad_batch; segment 0 = sr_recognise_batch). The reference only
// ever recognises segment 0 (main.c:268); here all <= 3 segments are (SURVEY 8f-3).
//
// One WARP per stream, built from the batch kernel's pieces (sr_vad_core.cuh): the new samples are appended to the
// stream's device row, the 80-sample blocks that became complete are summarised lane-parallel (16-byte loads, packed
// compares), the summaries are kept per stream, the frames that became complete are evaluated from them and the
// endpoint FSM is re-evaluated on the activity bitmap of the frames seen so far (a prefix of the capture yields exactly
// the decisions the sequential FSM has taken by then). One push = one H2D copy, five kernels whose batch sizes are read
// from device memory (no host round trip between VAD and recognition), one D2H copy, ONE synchronisation.
#include "sr_internal.h"
#include "sr_vad_core.cuh"
#include <condition_variable>
#include <deque>

namespace srk {

struct StreamState {            // one per stream, device resident
    atap_tag atap;
    u32 n;                      // samples received
    u32 blocks_done;            // 80-sample blocks summarised
    u32 word_base;              // frames < word_base are final (multiple of 32): their activity word is complete
    u32 cin_base;               // class of the last out-of-band sample in blocks < word_base (carried last_sig, VAD.C:99)
    u32 calibrated;
    u32 emitted;                // segments already reported
    u32 seg[6];
    u32 aw[32];                 // activity bitmap, frame f = bit f&31 of word f>>5 (<= 1024 frames: U <= 65535)
};

struct StreamEventDev {         // work list of the segments closed by the current push
    u32 stream, segment, start, end;
};

__global__ void stream_reset_kernel(StreamState *st, u32 S) {
    const u32 s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= S) return;
    StreamState z;
    memset(&z, 0, sizeof z);
    for (int i = 0; i < 6; ++i) z.seg[i] = SR_SEG_NULL;
    st[s] = z;
}

constexpr int kStreamWarps = 8;

// lens == NULL: every stream receives uniform_len samples; else stream s receives lens[s] (0 = nothing this time)
__global__ void __launch_bounds__(kStreamWarps * 32)
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
        const u16 *src = chunk + (size_t)s * chunk_stride;
        u16 *dst = x + n;
        if (((reinterpret_cast<uintptr_t>(src) | reinterpret_cast<uintptr_t>(dst)) & 15) == 0) {
            const u32 nv = len >> 3;
            for (u32 i = lane; i < nv; i += 32) reinterpret_cast<uint4 *>(dst)[i] = reinterpret_cast<const uint4 *>(src)[i];
            for (u32 i = 8 * nv + lane; i < len; i += 32) dst[i] = src[i];
        } else {
            for (u32 i = lane; i < len; i += 32) dst[i] = src[i];
        }
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
        if (n_len != 0 && n_len % 240u == 0) {                        // else atap stays untouched (VAD.C:33-36)
            u32 m, max_sum, abs_sum;
            atap_stats(x, vec_ok, n_len, lane, m, max_sum, abs_sum);
            atap_finish(at, n_len, m, max_sum, abs_sum);
        }
    }
    const u32 mid = at.mid_val, a_thl = mid + at.n_thl, b_thl = mid - at.n_thl;          // VAD.C:112-113 (u32 wrap)

    // frames i = 80k while i < L-160 (VAD.C:121) over the FINAL buffer length L; frame k = blocks k, k+1
    const u32 nfr_total = L > SR_FRAME_LEN ? (L - SR_FRAME_LEN + SR_FRAME_MOV - 1) / SR_FRAME_MOV : 0;
    const u32 nblk_total = nfr_total ? nfr_total + 1 : 0;
    const u32 nb_avail = min(n / 80u, nblk_total);

    // ---- summaries of the blocks that became complete -------------------------------------------------------------
    u32 blocks_done = sp->blocks_done;
    for (u32 blk0 = blocks_done; blk0 < nb_avail; blk0 += 32) {
        const u32 left = nb_avail - blk0;
        const u16 *xb = x + 80u * blk0;
        if (left <= 4u && (reinterpret_cast<uintptr_t>(xb) & 3) == 0) {            // few blocks: eight lanes per block
            u32 bs, fl;
            block_scan_split8(xb, lane, left, mid, a_thl, b_thl, bs, fl);
            const u32 blk = blk0 + (u32)(lane >> 3);
            if ((lane & 7) == 0 && blk < nb_avail) { info[2 * blk] = bs; info[2 * blk + 1] = fl; }
        } else if ((u32)lane < left) {
            VadWarpView v;
            v.x = xb; v.vec_ok = (reinterpret_cast<uintptr_t>(xb) & 15) == 0;
            u32 bs, fl;
            block_scan(v, 80u * (u32)lane, mid, a_thl, b_thl, bs, fl);
            info[2 * (blk0 + lane)] = bs; info[2 * (blk0 + lane) + 1] = fl;
        }
    }
    blocks_done = max(blocks_done, nb_avail);
    __syncwarp();

    // ---- frames that became complete: activity bitmap (the partial 32-frame word is simply re-evaluated) ------------
    const u32 ready = nb_avail ? min(nfr_total, nb_avail - 1u) : 0u;
    u32 aw = sp->aw[lane];
    u32 k0 = sp->word_base, cin = sp->cin_base;
    while (k0 < ready) {
        const u32 kend = min(ready, k0 + 32u);
        u32 c = cin;
        const u32 word = frames_pass(info, k0, kend, lane, at, c);
        if ((u32)lane == (k0 >> 5)) aw = word;
        if (kend != k0 + 32u) break;                                   // partial word: base and carry stay where they are
        cin = c; k0 += 32u;
    }

    // ---- endpoint FSM on the frames seen so far; report the segments that closed in this push -----------------------
    u32 seg[6] = {SR_SEG_NULL, SR_SEG_NULL, SR_SEG_NULL, SR_SEG_NULL, SR_SEG_NULL, SR_SEG_NULL};
    if (ready) fsm_segments(aw, ready, lane, seg);
    u32 emitted = sp->emitted;
    if (lane == 0) {
        for (u32 sgi = emitted; sgi < SR_MAX_VC_CON && seg[2 * sgi + 1] != SR_SEG_NULL; ++sgi) {
            const u32 e = atomicAdd(n_ev, 1u);
            if (e < cap) {
                StreamEventDev d; d.stream = s; d.segment = sgi; d.start = seg[2 * sgi]; d.end = seg[2 * sgi + 1];
                ev[e] = d;
                seg_ev[2 * e] = d.start; seg_ev[2 * e + 1] = d.end;
                atap_ev[e] = at; map_ev[e] = s;
            }
            ++emitted;
        }
        sp->atap = at; sp->n = n; sp->blocks_done = blocks_done; sp->word_base = k0; sp->cin_base = cin;
        sp->calibrated = calibrated; sp->emitted = emitted;
#pragma unroll
        for (int i = 0; i < 6; ++i) sp->seg[i] = seg[i];
    }
    sp->aw[lane] = aw;
}

__global__ void stream_segments_kernel(const StreamState *st, u32 S, u32 *seg_off, atap_tag *atap, u32 *n_recv) {
    const u32 s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= S) return;
    if (seg_off) for (int i = 0; i < 6; ++i) seg_off[(size_t)s * 6 + i] = st[s].seg[i];
    if (atap) atap[s] = st[s].atap;
    if (n_recv) n_recv[s] = st[s].n;
}

// status per event from the freshly computed features (MFCC fail = frm_num 0, main.c:269-274) + argmin initialiser
__global__ void stream_status_kernel(const unsigned char *ftr, const u32 *n_ev, u32 cap, u8 *status, u32 *frm, u64 *best) {
    const u32 i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= min(*n_ev, cap)) return;
    const u32 f = (*reinterpret_cast<const u32 *>(ftr + (size_t)i * kFtrBytes)) >> 16;
    status[i] = f == 0 ? SR_ST_MFCC_FAIL : SR_ST_OK;
    frm[i] = f;
    best[i] = ((u64)SR_DIS_MAX << 32) | 0ull;                        // main.c:276-278
}

// final argmin (main.c:285-294) + one packed record per event for a single D2H copy: word 0 of `out` = event count
__global__ void stream_finish_kernel(const StreamEventDev *ev, const u32 *n_ev, u32 cap, const u8 *status, const u32 *frm,
                                     const u64 *best, sr_stream_event *out_rec, u32 *out_count) {
    const u32 i = blockIdx.x * blockDim.x + threadIdx.x;
    const u32 ne = min(*n_ev, cap);
    if (i == 0) *out_count = ne;
    if (i >= ne) return;
    const u64 k = best[i];
    u32 idx = (u32)(k & 0xFFFFFFFFull), dis = (u32)(k >> 32);
    if (status[i] != SR_ST_OK) { idx = 0; dis = SR_DIS_ERR; }
    sr_stream_event r;
    r.stream = ev[i].stream; r.segment = ev[i].segment; r.start = ev[i].start; r.end = ev[i].end;
    r.status = status[i]; r.frm_num = frm[i]; r.best_idx = idx; r.best_dis = dis; r.cmd = idx / SR_FTR_PER_COMM;
    out_rec[i] = r;
}

}  // namespace srk

struct sr_stream_pool {
    sr_handle *h = nullptr;
    u32 S = 0, L = 0, n_len = 0, cap = 0, info_stride = 0, stage_stride = 0;
    DevBuf pcm, state, info, stage, lens, ev, seg_ev, atap_ev, map_ev, n_ev, ftr, status, frm, out;
    unsigned char *out_host = nullptr;             // pinned: [count u32, pad][records]
    u32 *lens_host = nullptr;                      // pinned staging of a ragged push's lengths
    std::deque<sr_stream_event> pending;           // events not yet handed to the caller (max_events too small)
    static constexpr u32 kQuick = 4096;            // records fetched with the count in the first D2H copy
};

static int streams_push_impl(sr_stream_pool *p, const uint16_t *chunk, uint32_t chunk_stride, uint32_t uniform_len,
                             const uint32_t *lens, sr_stream_event *events, uint32_t max_events, uint32_t *n_events);

extern "C" {

int sr_streams_destroy(sr_stream_pool *p) {
    if (!p) return 0;
    DeviceGuard g(p->h->device);
    cudaStreamSynchronize(p->h->stream);
    DevBuf *bufs[] = {&p->pcm, &p->state, &p->info, &p->stage, &p->lens, &p->ev, &p->seg_ev, &p->atap_ev, &p->map_ev,
                      &p->n_ev, &p->ftr, &p->status, &p->frm, &p->out};
    for (DevBuf *b : bufs) if (b->p) cudaFree(b->p);
    if (p->out_host) cudaFreeHost(p->out_host);
    if (p->lens_host) cudaFreeHost(p->lens_host);
    delete p;
    return 0;
}

int sr_streams_reset(sr_stream_pool *p) {
    SR_REQUIRE(nullptr, p != nullptr);
    sr_handle *h = p->h;
    DeviceGuard g(h->device);
    p->pending.clear();
    stream_reset_kernel<<<(p->S + 127) / 128, 128, 0, h->stream>>>(static_cast<StreamState *>(p->state.p), p->S);
    SR_CK(h, cudaGetLastError());
    SR_CK(h, cudaMemsetAsync(p->pcm.p, 0, (size_t)p->S * p->L * 2, h->stream));
    ++h->launches;
    return 0;
}

int sr_streams_create(sr_handle *h, uint32_t n_streams, uint32_t max_samples, uint32_t n_len, sr_stream_pool **out) {
    SR_REQUIRE(h, h && out && n_streams > 0 && max_samples > 0 && max_samples <= 65535u && n_len <= max_samples);
    DeviceGuard g(h->device);
    sr_stream_pool *p = new (std::nothrow) sr_stream_pool;
    SR_REQUIRE(h, p != nullptr);
    p->h = h; p->S = n_streams; p->L = max_samples; p->n_len = n_len; p->cap = 3 * n_streams;
    p->info_stride = 2 * (max_samples / 80 + 2);
    const size_t cap = p->cap;
    cudaError_t e = cudaSuccess;
    auto need = [&](DevBuf &b, size_t bytes) { if (e == cudaSuccess) e = ensure(b, bytes); };
    need(p->pcm, (size_t)n_streams * max_samples * 2 + 64);
    need(p->state, (size_t)n_streams * sizeof(StreamState));
    need(p->info, (size_t)n_streams * p->info_stride * 4);
    need(p->lens, (size_t)n_streams * 4);
    need(p->ev, cap * sizeof(StreamEventDev));
    need(p->seg_ev, cap * 8);
    need(p->atap_ev, cap * sizeof(atap_tag));
    need(p->map_ev, cap * 4);
    need(p->n_ev, 16);
    need(p->ftr, cap * kFtrBytes);
    need(p->status, cap);
    need(p->frm, cap * 4);
    need(p->out, 16 + cap * sizeof(sr_stream_event));
    if (e == cudaSuccess) e = cudaMallocHost(&p->out_host, 16 + cap * sizeof(sr_stream_event));
    if (e == cudaSuccess) e = cudaMallocHost(&p->lens_host, (size_t)n_streams * 4);
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
    u32 k = 0;
    while (k < max_events && events && !p->pending.empty()) { events[k++] = p->pending.front(); p->pending.pop_front(); }
    *n_events = k;
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
    stream_segments_kernel<<<(p->S + 127) / 128, 128, 0, h->stream>>>(static_cast<const StreamState *>(p->state.p), p->S,
                                                                     static_cast<u32 *>(h->seg.p), static_cast<atap_tag *>(h->atap.p), nullptr);
    SR_CK(h, cudaGetLastError());
    ++h->launches;
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
    u32 max_len = uniform_len;
    if (lens) {
        max_len = 0;
        for (u32 s = 0; s < p->S; ++s) { p->lens_host[s] = lens[s]; if (lens[s] > max_len) max_len = lens[s]; }
    }
    SR_REQUIRE(h, max_len == 0 || chunk != nullptr);
    SR_REQUIRE(h, max_len <= p->L && chunk_stride >= max_len);
    DeviceGuard g(h->device);
    if (h->comm) { const int rc = sr_comm_wait(h); if (rc) return rc; }   // a pending gather may still read the handle's key buffer
    const u16 *chunk_dev = static_cast<const u16 *>(p->stage.p);
    u32 chunk_dev_stride = p->stage_stride;
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
            SR_CK(h, ensure(p->stage, (size_t)p->S * sstride * 2 + 64));
            p->stage_stride = sstride;
            chunk_dev = static_cast<const u16 *>(p->stage.p); chunk_dev_stride = sstride;
            SR_CK(h, cudaMemcpy2DAsync(p->stage.p, (size_t)sstride * 2, chunk, (size_t)chunk_stride * 2, (size_t)max_len * 2, p->S,
                                       cudaMemcpyHostToDevice, h->stream));
        }
        if (lens) SR_CK(h, cudaMemcpyAsync(p->lens.p, p->lens_host, (size_t)p->S * 4, cudaMemcpyHostToDevice, h->stream));
    }
    SR_CK(h, cudaMemsetAsync(p->n_ev.p, 0, 4, h->stream));
    u32 *n_ev = static_cast<u32 *>(p->n_ev.p);
    stream_step_kernel<<<(p->S + kStreamWarps - 1) / kStreamWarps, kStreamWarps * 32, 0, h->stream>>>(
        static_cast<u16 *>(p->pcm.p), p->L, p->S, chunk_dev, chunk_dev_stride, max_len ? uniform_len : 0u,
        (lens && max_len) ? static_cast<const u32 *>(p->lens.p) : nullptr, p->n_len, static_cast<StreamState *>(p->state.p),
        static_cast<u32 *>(p->info.p), p->info_stride, static_cast<StreamEventDev *>(p->ev.p), static_cast<u32 *>(p->seg_ev.p),
        static_cast<atap_tag *>(p->atap_ev.p), static_cast<u32 *>(p->map_ev.p), n_ev, p->cap);
    SR_CK(h, cudaGetLastError());
    // recognise the closed segments; every kernel reads the number of events from device memory (upper bound: cap)
    SR_CK(h, launch_mfcc_h(h, static_cast<const u16 *>(p->pcm.p), p->L, p->cap, static_cast<const u32 *>(p->seg_ev.p), 2,
                           static_cast<const atap_tag *>(p->atap_ev.p), p->ftr.p, static_cast<const u32 *>(p->map_ev.p), p->S, n_ev));
    SR_CK(h, ensure(h->best, (size_t)p->cap * 8));
    u64 *best = static_cast<u64 *>(h->best.p);
    const u32 gb = (p->cap + 255) / 256;
    stream_status_kernel<<<gb, 256, 0, h->stream>>>(static_cast<const unsigned char *>(p->ftr.p), n_ev, p->cap,
                                                   static_cast<u8 *>(p->status.p), static_cast<u32 *>(p->frm.p), best);
    SR_CK(h, cudaGetLastError());
    if (h->n_slot)
        SR_CK(h, launch_dtw_h(h, p->ftr.p, p->cap, SR_DTW_CHECK_SIGN, nullptr, best, static_cast<const u8 *>(p->status.p), n_ev));
    u32 *out_count = static_cast<u32 *>(p->out.p);
    sr_stream_event *out_rec = reinterpret_cast<sr_stream_event *>(static_cast<unsigned char *>(p->out.p) + 16);
    stream_finish_kernel<<<gb, 256, 0, h->stream>>>(static_cast<const StreamEventDev *>(p->ev.p), n_ev, p->cap,
                                                   static_cast<const u8 *>(p->status.p), static_cast<const u32 *>(p->frm.p),
                                                   best, out_rec, out_count);
    SR_CK(h, cudaGetLastError());
    h->launches += 4 + (h->n_slot ? 1 : 0);
    const u32 quick = p->cap < sr_stream_pool::kQuick ? p->cap : sr_stream_pool::kQuick;
    D2H(h, p->out_host, p->out.p, 16 + (size_t)quick * sizeof(sr_stream_event));
    SR_CK(h, cudaStreamSynchronize(h->stream));                       // the one synchronisation of a push
    const u32 ne = *reinterpret_cast<const u32 *>(p->out_host);
    if (ne > quick) {                                                 // rare: a burst of closings larger than the quick window
        D2H(h, p->out_host + 16 + (size_t)quick * sizeof(sr_stream_event), static_cast<unsigned char *>(p->out.p) + 16 + (size_t)quick * sizeof(sr_stream_event),
            (size_t)(ne - quick) * sizeof(sr_stream_event));
        SR_CK(h, cudaStreamSynchronize(h->stream));
    }
    const sr_stream_event *rec = reinterpret_cast<const sr_stream_event *>(p->out_host + 16);
    u32 k = 0;
    // older queued events first, then this push's; whatever does not fit stays queued for sr_streams_fetch
    while (k < max_events && events && !p->pending.empty()) { events[k++] = p->pending.front(); p->pending.pop_front(); }
    u32 i = 0;
    if (p->pending.empty()) for (; i < ne && k < max_events && events; ++i) events[k++] = rec[i];
    for (; i < ne; ++i) p->pending.push_back(rec[i]);
    *n_events = k;
    return 0;
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
    if (!handles || !out || n_handles == 0 || n_streams < n_handles) return fail(nullptr, "sr_stream_group_create: bad arguments", cudaSuccess);
    sr_stream_group *gr = new (std::nothrow) sr_stream_group;
    if (!gr) return fail(nullptr, "sr_stream_group_create: out of memory", cudaErrorMemoryAllocation);
    gr->S = n_streams;
    for (u32 g = 0; g < n_handles; ++g) {
        auto *sh = new sr_stream_group::Shard;
        sh->s0 = (u32)((uint64_t)n_streams * g / n_handles);
        sh->S = (u32)((uint64_t)n_streams * (g + 1) / n_handles) - sh->s0;
        gr->shards.push_back(sh);
        const int rc = sr_streams_create(handles[g], sh->S, max_samples, n_len, &sh->pool);
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
