// sr_api.cu -- the C-ABI of libspeech_b200.so (include/speech_recog.h): handle, device workspaces,
// host<->device plumbing and the reference-named batch-of-1 entry points. No arithmetic of the
// recognition path happens on the host: every result is produced by the kernels in sr_vad.cu,
// sr_mfcc.cu and sr_dtw.cu. Without a CUDA device every entry point fails loudly.
#include "sr_internal.h"
#include "../../include/sr_synth.h"
#include "sr_pack_host.h"
#include "sr_numa.h"
#include <map>
#include <algorithm>
#include <type_traits>

static int device_numa_node(int device) {
    char id[64] = {0};
    if (cudaDeviceGetPCIBusId(id, (int)sizeof id, device) != cudaSuccess) { cudaGetLastError(); return -1; }
    return numa_node_of_pci(id);
}

extern "C" {

int sr_abi_version(void) { return 12; }

int sr_device_count(void) {
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess) { cudaGetLastError(); return 0; }
    return n;
}

const char *sr_last_error(const sr_handle *h) { return h ? h->err.c_str() : g_tls_error.c_str(); }

int sr_create(int device, sr_handle **out) {
    if (!out) return fail(nullptr, "sr_create: out == NULL", cudaSuccess);
    *out = nullptr;
    int n = 0;
    cudaError_t e = cudaGetDeviceCount(&n);
    if (e != cudaSuccess || n == 0)
        return fail(nullptr, "sr_create: no CUDA device (libspeech_b200 has no CPU fallback)", e == cudaSuccess ? cudaErrorNoDevice : e);
    if (device < 0) SR_CK(nullptr, cudaGetDevice(&device));
    if (device >= n) return fail(nullptr, "sr_create: device ordinal out of range", cudaErrorInvalidDevice);
    sr_handle *h = new (std::nothrow) sr_handle;
    if (!h) return fail(nullptr, "sr_create: out of host memory", cudaErrorMemoryAllocation);
    h->device = device;
    DeviceGuard g(device);
    if (!g.ok) { delete h; return fail(nullptr, "sr_create: cudaSetDevice", cudaErrorInvalidDevice); }
    cudaDeviceProp prop;
    e = cudaGetDeviceProperties(&prop, device);
    if (e != cudaSuccess) { delete h; return fail(nullptr, "cudaGetDeviceProperties", e); }
    if (prop.major != 9 || prop.minor != 0) {           // sm_90a code runs on compute capability 9.0 only
        delete h;
        return fail(nullptr, "sr_create: kernels are built for sm_90a (H100) only", cudaErrorInvalidDevice);
    }
    h->num_sms = prop.multiProcessorCount;
    h->numa_node = device_numa_node(device);
    // every failure from here on goes through sr_destroy, which releases whatever has been created so far
    e = cudaStreamCreateWithFlags(&h->own_stream, cudaStreamNonBlocking);
    h->stream = h->own_stream;
    if (e == cudaSuccess) e = cudaStreamCreateWithFlags(&h->copy_stream, cudaStreamNonBlocking);
    for (int i = 0; i < 2 && e == cudaSuccess; ++i) {
        e = cudaEventCreateWithFlags(&h->ev_h2d[i], cudaEventDisableTiming | cudaEventBlockingSync);   // the packed transport's sender sleeps on it
        if (e == cudaSuccess) e = cudaEventCreateWithFlags(&h->ev_done[i], cudaEventDisableTiming);
    }
    if (e != cudaSuccess) { sr_destroy(h); return fail(nullptr, "sr_create: stream/event creation", e); }
    if (!dev_tables()) { sr_destroy(h); return fail(nullptr, "sr_create: table upload", cudaErrorInitializationError); }
    *out = h;
    return 0;
}

int sr_destroy(sr_handle *h) {
    if (!h) return 0;
    DeviceGuard g(h->device);
    if (h->stream) cudaStreamSynchronize(h->stream);
    sr_comm_destroy(h);
    for (cudaEvent_t e : h->ev) cudaEventDestroy(e);
    if (h->own_stream) cudaStreamDestroy(h->own_stream);
    if (h->copy_stream) cudaStreamDestroy(h->copy_stream);
    for (int i = 0; i < 2; ++i) { if (h->ev_h2d[i]) cudaEventDestroy(h->ev_h2d[i]); if (h->ev_done[i]) cudaEventDestroy(h->ev_done[i]); }
    delete h;                                           // frees the workspaces and stops the transport's workers, under g
    return 0;
}

int sr_set_stream(sr_handle *h, void *cuda_stream) {
    SR_REQUIRE(h, h != nullptr);
    h->stream = static_cast<cudaStream_t>(cuda_stream);     // used verbatim: NULL is CUDA's legacy default stream
    return 0;
}

int sr_use_own_stream(sr_handle *h) {
    SR_REQUIRE(h, h != nullptr);
    h->stream = h->own_stream;
    return 0;
}

int sr_sync(sr_handle *h) {
    SR_REQUIRE(h, h != nullptr);
    DeviceGuard g(h->device);
    if (h->comm) { const int rc = sr_comm_wait(h); if (rc) return rc; }   // collectives issued so far are covered too
    SR_CK(h, cudaStreamSynchronize(h->stream));
    return 0;
}

int sr_set_geometry(sr_handle *h, int geom) {
    SR_REQUIRE(h, h && (geom == SR_GEOM_REF || geom == SR_GEOM_B));
    h->geom = geom;
    return 0;
}
int sr_get_geometry(const sr_handle *h) { return h ? h->geom : SR_GEOM_REF; }

int sr_set_dtw_variant(sr_handle *h, int variant) {
    SR_REQUIRE(h, h && variant >= -1 && variant <= 1);
    h->dtw_variant = variant;
    return 0;
}

int sr_set_match(sr_handle *h, uint32_t flags, int band_r) {
    // the matcher, the lifter and the decision rules; the recognition calls add SR_DTW_CHECK_SIGN themselves
    ScanPlan p;
    SR_REQUIRE(h, h && !(flags & SR_DTW_CHECK_SIGN) && scan_plan(flags, band_r, 0, true, &p));
    h->match_flags = flags;
    h->match_r = band_r;
    return 0;
}
int sr_get_match(const sr_handle *h, uint32_t *flags, int *band_r) {
    if (!h || !flags || !band_r) return fail(nullptr, "sr_get_match: bad arguments", cudaSuccess);
    *flags = h->match_flags;
    *band_r = h->match_r;
    return 0;
}

uint64_t sr_launch_count(const sr_handle *h) { return h ? h->launches : 0; }

// ---- pinned host memory -------------------------------------------------------------------------------
// sr_host_alloc_dev places the pages on the NUMA node the GPU hangs off (first touch on that node's CPUs, then
// cudaHostRegister), so the H2D copy never crosses the socket interconnect; sr_host_alloc is the plain form.
static std::mutex g_host_mu;
static std::map<void *, size_t> g_node_allocs;           // node_alloc'ed + registered regions -> length

int sr_device_numa_node(int device) {
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess || device < 0 || device >= n) { cudaGetLastError(); return -1; }
    return device_numa_node(device);
}

int sr_bind_thread_to_device(int device) {
    const int node = sr_device_numa_node(device);
    cpu_set_t want;
    if (node < 0 || numa_node_count() < 2 || !cpus_of_node(node, &want)) return -1;
    if (sched_setaffinity(0, sizeof want, &want) != 0) return -1;
    return node;
}

void *sr_host_alloc(size_t bytes) {
    void *p = nullptr;
    if (cudaMallocHost(&p, bytes) != cudaSuccess) { cudaGetLastError(); return nullptr; }
    return p;
}

void *sr_host_alloc_dev(int device, size_t bytes) {
    if (bytes == 0) return nullptr;
    const int node = sr_device_numa_node(device);
    if (node < 0 || numa_node_count() < 2) return sr_host_alloc(bytes);     // single node: nothing to place
    void *p = node_alloc(bytes, node);
    if (!p) return nullptr;
    if (cudaHostRegister(p, bytes, cudaHostRegisterPortable) != cudaSuccess) { cudaGetLastError(); node_free(p, bytes); return nullptr; }
    std::lock_guard<std::mutex> lk(g_host_mu);
    g_node_allocs[p] = bytes;
    return p;
}

void sr_host_free(void *p) {
    if (!p) return;
    size_t bytes = 0;
    {
        std::lock_guard<std::mutex> lk(g_host_mu);
        auto it = g_node_allocs.find(p);
        if (it != g_node_allocs.end()) { bytes = it->second; g_node_allocs.erase(it); }
    }
    if (bytes) { cudaHostUnregister(p); node_free(p, bytes); }
    else cudaFreeHost(p);
}

int sr_host_numa_node(const void *p) { return p ? numa_node_of_page(p) : -1; }

// ---- kernel launches (launch_on, sr_internal.h) --------------------------------------------------------------------
int sr_timing_enable(sr_handle *h, uint32_t max_records) {
    SR_REQUIRE(h, h != nullptr);
    DeviceGuard g(h->device);
    for (cudaEvent_t e : h->ev) cudaEventDestroy(e);
    h->ev.clear(); h->ev_tag.clear(); h->ev_used = 0;
    h->timing = max_records > 0;
    for (uint32_t i = 0; i < 2 * max_records; ++i) {
        cudaEvent_t e;
        SR_CK(h, cudaEventCreate(&e));
        h->ev.push_back(e);
    }
    h->ev_tag.assign(max_records, 0);
    return 0;
}
int sr_timing_collect(sr_handle *h, uint32_t *tags, float *ms, uint32_t cap, uint32_t *n) {
    SR_REQUIRE(h, h && n);
    DeviceGuard g(h->device);
    SR_CK(h, cudaStreamSynchronize(h->stream));
    uint32_t k = 0;
    for (size_t i = 0; i < h->ev_used && k < cap; ++i, ++k) {
        float t = 0.f;
        SR_CK(h, cudaEventElapsedTime(&t, h->ev[2 * i], h->ev[2 * i + 1]));
        if (tags) tags[k] = h->ev_tag[i];
        if (ms) ms[k] = t;
    }
    *n = k;
    h->ev_used = 0;
    return 0;
}

}  // extern "C"

// get_mfcc (MFCC.C) and get_mdl (DTW.C) never write save_sign: copy back bytes [2, 2860) of each of n structs only
static cudaError_t ftr_to_host(sr_handle *h, v_ftr_tag *dst, const void *src, size_t n) {
    return cudaMemcpy2DAsync(reinterpret_cast<unsigned char *>(dst) + 2, kFtrBytes, static_cast<const unsigned char *>(src) + 2,
                             kFtrBytes, kFtrBytes - 2, n, cudaMemcpyDeviceToHost, h->stream);
}

// the captures of a host-buffer call: 1..65 535 samples each, the calibration window inside them
static bool capture_args_ok(u32 U, u32 B, u32 n_len) { return (B == 0 || U > 0) && U <= 65535u && n_len <= U; }

// the B atap records noise_atap runs on: the caller's (atap != NULL), else B zeroed ones in w
static cudaError_t atap_or_zeroed(sr_handle *h, DevBuf &w, u32 B, atap_tag *&atap) {
    if (atap) return cudaSuccess;
    const cudaError_t e = ensure(w, (size_t)B * sizeof(atap_tag), atap);
    return e != cudaSuccess ? e : cudaMemsetAsync(atap, 0, (size_t)B * sizeof(atap_tag), h->stream);
}

// One host-buffer call: inputs staged into handle workspaces, kernels, outputs copied back, one synchronisation. The
// first failure is kept (its message prefixed with the call's name) and every later step is skipped; finish() returns it.
struct HostCall {
    sr_handle *h;
    const char *name;
    DeviceGuard g;
    int rc = 0;
    struct Back { void *dst; const void *src; size_t bytes; bool ftr; };
    std::vector<Back> back;

    HostCall(sr_handle *hh, const char *nm) : h(hh), name(nm), g(hh->device) {}
    void took(int r) {
        if (!r || rc) return;
        rc = r;
        h->err = std::string(name) + ": " + h->err;
        g_tls_error = h->err;
    }
    void ck(const char *what, cudaError_t e) { if (!rc && e != cudaSuccess) took(fail(h, what, e)); }
    template <class F> void run(F f) { if (!rc) took(f()); }
    template <class F> void launch(int tag, const char *what, F f) { if (!rc) took(launch_on(h, tag, what, f)); }
    // workspace w, at least `bytes` long (NULL once the call has failed)
    template <class T = void> T *ws(DevBuf &w, size_t bytes) {
        if (!rc) ck("ensure", ensure(w, bytes));
        return rc ? nullptr : static_cast<T *>(w.p);
    }
    void h2d(void *dst, const void *src, size_t bytes) {
        if (!rc && bytes) ck("cudaMemcpyAsync host->device", cudaMemcpyAsync(dst, src, bytes, cudaMemcpyHostToDevice, h->stream));
    }
    // `bytes` of host input src staged in workspace w (slack: extra bytes the kernel may read past the end)
    template <class T> T *in(DevBuf &w, const T *src, size_t bytes, size_t slack = 0) {
        T *d = ws<T>(w, bytes + slack);
        h2d(d, src, bytes);
        return d;
    }
    // workspace w for an output that finish() copies back to dst (if dst != NULL); v_ftr_tag outputs skip save_sign
    template <class T> T *out(DevBuf &w, T *dst, size_t bytes, size_t slack = 0) {
        T *d = ws<T>(w, bytes + slack);
        if (d && dst && bytes) back.push_back({dst, d, bytes, std::is_same_v<T, v_ftr_tag>});
        return d;
    }
    // B atap records in w (atap_or_zeroed): the caller's host records staged in -- and copied back when `back`: noise_atap
    // leaves them untouched when n_len % 240 != 0 -- or zeroed ones when src is NULL
    atap_tag *atap(DevBuf &w, atap_tag *src, u32 B, bool back) {
        const size_t bytes = (size_t)B * sizeof(atap_tag);
        atap_tag *d = src ? in(w, src, bytes) : nullptr;
        if (src && back) out(w, src, bytes);
        if (!src && !rc) ck("atap_or_zeroed", atap_or_zeroed(h, w, B, d));
        return rc ? nullptr : d;
    }
    int finish() {
        for (const Back &b : back)
            ck("copy back", b.ftr ? ftr_to_host(h, static_cast<v_ftr_tag *>(b.dst), b.src, b.bytes / kFtrBytes)
                                  : cudaMemcpyAsync(b.dst, b.src, b.bytes, cudaMemcpyDeviceToHost, h->stream));
        ck("cudaStreamSynchronize", cudaStreamSynchronize(h->stream));
        return rc;
    }
};

// Host PCM [B][U] of the host call c sent to the device in n groups of G recordings (the last one fewer) through the two
// buffers of h->pcm: with more than one group, the copy of the next group (copy stream) overlaps the kernels of this one
// (compute stream).
struct PcmGroups {
    sr_handle *h;
    u32 G, n;
    size_t bytes;                                       // one buffer: G recordings, 256-byte aligned
    PcmGroups(HostCall &c, u32 U, u32 B, u32 g) : h(c.h), G(g), n((B + g - 1) / g), bytes((((size_t)g * U * 2 + 255) / 256) * 256) {
        c.ws(h->pcm, (n > 1 ? 2 : 1) * bytes + 16);
    }
    u16 *buf(int i) const { return reinterpret_cast<u16 *>(static_cast<unsigned char *>(h->pcm.p) + (size_t)i * bytes); }
    // the k-th group sent, into buffer k & 1: once the kernels of group k - 2 are done with it, `size` bytes from src to dst,
    // then the compute stream waits for the copy
    cudaError_t send(u32 k, void *dst, const void *src, size_t size) const {
        if (n == 1) return cudaMemcpyAsync(dst, src, size, cudaMemcpyHostToDevice, h->stream);
        cudaError_t e = k >= 2 ? cudaStreamWaitEvent(h->copy_stream, h->ev_done[k & 1], 0) : cudaSuccess;
        if (e == cudaSuccess) e = cudaMemcpyAsync(dst, src, size, cudaMemcpyHostToDevice, h->copy_stream);
        if (e == cudaSuccess) e = cudaEventRecord(h->ev_h2d[k & 1], h->copy_stream);
        if (e == cudaSuccess) e = cudaStreamWaitEvent(h->stream, h->ev_h2d[k & 1], 0);
        return e;
    }
    // after the kernels of the k-th group: its buffer is free again
    cudaError_t done(u32 k) const { return n > 1 ? cudaEventRecord(h->ev_done[k & 1], h->stream) : cudaSuccess; }
};

// ---- input at another rate (include/sr_synth.h) ------------------------------------------------------------------------
static const ResampleRate kRate8k{8000, 1, 1, 1, 0};

// ceil(n * L / M): the 8 kHz samples K15 makes of n input samples at the rate r
static uint64_t rate_len(uint64_t n, const ResampleRate &r) { return (n * r.L + r.M - 1) / r.M; }

// the argument rules of a capture call at a rate: the rate, and the 8 kHz call's rules with U8 = ceil(U_in * L / M) for U
static bool capture_rate_args_ok(uint32_t rate, u32 U_in, u32 B, u32 n_len, ResampleRate *r) {
    if (!resample_rate(rate, r)) return false;
    const uint64_t U8 = rate_len(U_in, *r);
    return U8 <= 65535u && capture_args_ok((u32)U8, B, n_len);
}

// The B captures of a whole-batch capture call staged in one copy, as the 8 kHz body reads them: at 8 kHz the caller's
// rows in pcm. At another rate the rows of U_in samples go to pcm, then one K15 launch (tag 15) writes rows of
// U8 = ceil(U_in * L / M) samples to pcm8, and the body reads those. Both carry the 16 bytes of slack of the 8 kHz staging.
// K15's grid (B * tiles < 2^31, at most 32 tiles of 2 048 outputs per capture) holds for any batch whose features fit
// device memory; a larger one fails at the launch.
static const u16 *stage_captures(HostCall &c, const uint16_t *pcm, u32 U_in, u32 B, const ResampleRate &r) {
    sr_handle *h = c.h;
    const u16 *d_pcm = c.in(h->pcm, pcm, (size_t)B * U_in * 2, 16);
    if (r.rate == 8000) return d_pcm;
    const u32 U8 = (u32)rate_len(U_in, r);
    u16 *d_pcm8 = c.ws<u16>(h->pcm8, (size_t)B * U8 * 2 + 16);
    c.launch(TAG_RESAMPLE, "launch_resample_adc12", [&] {
        return launch_resample_adc12(d_pcm, U_in, B, nullptr, r.rate, d_pcm8, U8, nullptr, h->device, h->stream);
    });
    return d_pcm8;
}

extern "C" {

// ---- template bank --------------------------------------------------------------------------------
// Banks wider than one 32-template tile are walked in ascending frm_num order, so that the templates sharing a warp have
// similar walk lengths (CPU model: mean/max walk length per tile 0.81 -> 0.88 at T = 200). The order is a hint: scores and
// argmin keys carry the original slot numbers, and a stale order (bank rewritten in place) only costs efficiency.
static int bank_order(sr_handle *h, const unsigned char *hdr_host /* n_slot headers, 4 bytes each, or NULL: fetch */) {
    BankView &b = h->bank;
    b.order = nullptr;
    const u32 T = b.n;
    if (T <= 32 || !b.p) { h->perm_bank = b.p; h->perm_n = T; h->perm_stride = b.stride; return 0; }
    std::vector<u32> hdr(T);
    if (hdr_host) memcpy(hdr.data(), hdr_host, (size_t)T * 4);
    else {
        SR_CK(h, cudaMemcpy2DAsync(hdr.data(), 4, b.p, b.stride, 4, T, cudaMemcpyDeviceToHost, h->stream));
        SR_CK(h, cudaStreamSynchronize(h->stream));
    }
    std::vector<u32> order(T);
    for (u32 i = 0; i < T; ++i) order[i] = i;
    auto key = [&](u32 i) { const u32 f = hdr[i] >> 16; return f > 119u ? 0xFFFFu : f; };   // garbage headers last
    std::stable_sort(order.begin(), order.end(), [&](u32 a, u32 c) { return key(a) < key(c); });
    SR_CK(h, ensure(h->bank_perm, (size_t)T * 4));
    SR_CK(h, cudaMemcpyAsync(h->bank_perm.p, order.data(), (size_t)T * 4, cudaMemcpyHostToDevice, h->stream));
    SR_CK(h, cudaStreamSynchronize(h->stream));                     // `order` is a local
    b.order = static_cast<const u32 *>(h->bank_perm.p);
    h->perm_bank = b.p; h->perm_n = T; h->perm_stride = b.stride;
    return 0;
}

int sr_set_bank_dev(sr_handle *h, const void *bank_dev, uint32_t n_slot, uint32_t slot_stride) {
    SR_REQUIRE(h, h != nullptr);
    SR_REQUIRE(h, n_slot == 0 || (bank_dev != nullptr && slot_stride >= (uint32_t)kFtrBytes && slot_stride % 4 == 0));
    SR_REQUIRE(h, (reinterpret_cast<uintptr_t>(bank_dev) & 3) == 0);
    const bool same = h->perm_bank == bank_dev && h->perm_n == n_slot && h->perm_stride == slot_stride;
    h->bank = {bank_dev, n_slot, slot_stride, h->bank.order};
    if (same) return 0;                                   // same buffer as last time (callers re-set it per batch): keep the order
    DeviceGuard g(h->device);
    return bank_order(h, nullptr);
}
int sr_set_bank(sr_handle *h, const void *bank, uint32_t n_slot, uint32_t slot_stride) {
    SR_REQUIRE(h, h != nullptr);
    SR_REQUIRE(h, n_slot == 0 || (bank != nullptr && slot_stride >= (uint32_t)kFtrBytes && slot_stride % 4 == 0));
    DeviceGuard g(h->device);
    const size_t bytes = (size_t)n_slot * slot_stride;
    SR_CK(h, cudaStreamSynchronize(h->stream));
    SR_CK(h, ensure(h->bank_own, bytes + 16));
    if (bytes) SR_CK(h, cudaMemcpyAsync(h->bank_own.p, bank, bytes, cudaMemcpyHostToDevice, h->stream));
    SR_CK(h, cudaStreamSynchronize(h->stream));
    h->bank = {h->bank_own.p, n_slot, slot_stride, nullptr};
    std::vector<u32> hdr(n_slot);
    for (u32 i = 0; i < n_slot; ++i) memcpy(&hdr[i], static_cast<const unsigned char *>(bank) + (size_t)i * slot_stride, 4);
    return bank_order(h, reinterpret_cast<const unsigned char *>(hdr.data()));
}

// ---- command labels: commstr[] of main.c:25-31, what spch_recg returns (main.c:295) ---------------------------------
// default table = the reference's own 18 entries: "0 " .. "9 " and the GBK codes of up/down/front/back/left/right/big/small
static const uint8_t kRefLabels[18][3] = {
    {0x30, 0x20, 0}, {0x31, 0x20, 0}, {0x32, 0x20, 0}, {0x33, 0x20, 0}, {0x34, 0x20, 0}, {0x35, 0x20, 0}, {0x36, 0x20, 0},
    {0x37, 0x20, 0}, {0x38, 0x20, 0}, {0x39, 0x20, 0}, {0xC9, 0xCF, 0}, {0xCF, 0xC2, 0}, {0xC7, 0xB0, 0}, {0xBA, 0xF3, 0},
    {0xD7, 0xF3, 0}, {0xD3, 0xD2, 0}, {0xB4, 0xF3, 0}, {0xD0, 0xA1, 0}};

int sr_set_labels(sr_handle *h, const void *labels, uint32_t n_labels, uint32_t label_stride) {
    SR_REQUIRE(h, h && (n_labels == 0 || (labels && label_stride > 0)));
    h->labels.assign(static_cast<const uint8_t *>(labels), static_cast<const uint8_t *>(labels) + (size_t)n_labels * label_stride);
    h->n_labels = n_labels; h->label_stride = label_stride;
    return 0;
}

const uint8_t *sr_label(const sr_handle *h, uint32_t cmd) {
    if (h && h->label_stride) return cmd < h->n_labels ? h->labels.data() + (size_t)cmd * h->label_stride : nullptr;
    return cmd < 18u ? kRefLabels[cmd] : nullptr;                  // no table set: the reference's
}

int sr_labels_batch(const sr_handle *h, const uint32_t *cmd, const uint8_t *status, uint32_t B, const uint8_t **labels_out) {
    if (!cmd || !labels_out) return -1;
    for (uint32_t b = 0; b < B; ++b)                               // NULL = spch_recg's early returns (main.c:261-274)
        labels_out[b] = (status && status[b] != SR_ST_OK) ? nullptr : sr_label(h, cmd[b]);
    return 0;
}

// ---- device-pointer entry points ------------------------------------------------------------------
int sr_noise_atap_batch_dev(sr_handle *h, const uint16_t *pcm, uint32_t U, uint32_t B, uint32_t n_len, atap_tag *atap) {
    SR_REQUIRE(h, h && (B == 0 || (pcm && atap)));
    SR_REQUIRE(h, U <= 65535u && n_len <= 65535u);
    if (B == 0) return 0;
    DeviceGuard g(h->device);
    SR_LAUNCH(h, TAG_VAD, launch_vad(pcm, U, B, n_len, 0, 1, 0, atap, nullptr, h->num_sms, h->stream, vad_work(h)));
    return 0;
}

int sr_vad_batch_dev(sr_handle *h, const uint16_t *pcm, uint32_t U, uint32_t B, uint32_t buf_len, const atap_tag *atap,
                     uint32_t *seg_off) {
    SR_REQUIRE(h, h && (B == 0 || (pcm && atap && seg_off)));
    SR_REQUIRE(h, U <= 65535u && buf_len <= U);
    if (B == 0) return 0;
    DeviceGuard g(h->device);
    SR_LAUNCH(h, TAG_VAD, launch_vad(pcm, U, B, 0, buf_len, 0, 1, const_cast<atap_tag *>(atap), seg_off, h->num_sms, h->stream, vad_work(h)));
    return 0;
}

int sr_mfcc_batch_dev(sr_handle *h, const uint16_t *pcm, uint32_t U, uint32_t B, const uint32_t *seg, uint32_t seg_stride,
                      const atap_tag *atap, v_ftr_tag *ftr) {
    SR_REQUIRE(h, h && (B == 0 || (pcm && seg && atap && ftr)));
    SR_REQUIRE(h, seg_stride >= 2 && (reinterpret_cast<uintptr_t>(ftr) & 3) == 0);
    if (B == 0) return 0;
    DeviceGuard g(h->device);
    SR_LAUNCH(h, TAG_MFCC, launch_mfcc_h(h, pcm, U, B, seg, seg_stride, atap, ftr));
    return 0;
}

}  // extern "C"

// main.c:276-291 on n inputs (n_dev: n on the device) under plan p: w's n argmin keys, then under a decision rule
// (p.rule.C > 0) n * C keys, set to their start (tag 3), and the template scan into them (p.tag); no w: it writes scores
// only
static int scan_to_keys(sr_handle *h, DevBuf *w, const ScanPlan &p, const BankView &bank, const void *in, u32 n, u32 *score,
                        const u8 *status, u64 *&keys, const u32 *n_dev = nullptr) {
    const u32 C = p.rule.C;
    keys = nullptr;
    if (w) {
        SR_CK(h, ensure(*w, (size_t)n * (1 + C) * 8));
        keys = static_cast<u64 *>(w->p) + (C ? n : 0);
        SR_LAUNCH(h, TAG_BEST_INIT, launch_best_init(keys, (u64)n * (C ? C : 1), h->stream));
    }
    if (bank.n) SR_LAUNCH(h, p.tag, launch_scan(h, p, scan_args(p, bank, in, n, score, keys, status, n_dev)));
    return 0;
}

// the template scan of B inputs against `bank`, then the argmin of each when one of best_idx / best_dis / cmd is wanted.
// With a status (the recognition calls) the flags may carry a decision rule, and the status is an output of its decision
// too; without one (sr_dtw_batch*) they may not.
static int dtw_dev_impl(sr_handle *h, const BankView &bank, const v_ftr_tag *in, uint32_t B, uint32_t flags, int band_r,
                        uint32_t *score, uint32_t *best_idx, uint32_t *best_dis, uint32_t *cmd, const u8 *status) {
    SR_REQUIRE(h, h && (B == 0 || in));
    SR_REQUIRE(h, (reinterpret_cast<uintptr_t>(in) & 3) == 0);
    ScanPlan p;                                                             // no input: no template is scanned
    SR_REQUIRE(h, scan_plan(flags, band_r, B ? bank.n : 0, status != nullptr, &p));
    if (B == 0) return 0;
    const bool want_best = best_idx || best_dis || cmd || p.rule.C;
    DevBuf &bb = key_buf(h);
    u64 *keys;
    if (const int rc = scan_to_keys(h, want_best ? &bb : nullptr, p, bank, in, B, score, status, keys)) return rc;
    u64 *best = static_cast<u64 *>(bb.p);
    if (want_best)
        SR_LAUNCH(h, TAG_BEST_FINAL, launch_best_final(best, keys, B, p.rule, best_idx, best_dis, cmd, const_cast<u8 *>(status),
                                                       h->stream));
    return 0;
}

extern "C" int sr_dtw_batch_dev(sr_handle *h, const v_ftr_tag *in, uint32_t B, uint32_t flags, int band_r, uint32_t *score,
                                uint32_t *best_idx, uint32_t *best_dis) {
    SR_REQUIRE(h, h != nullptr);
    DeviceGuard g(h->device);
    return dtw_dev_impl(h, h->bank, in, B, flags, band_r, score, best_idx, best_dis, nullptr, nullptr);
}

extern "C" int sr_recognise_batch_dev(sr_handle *h, const uint16_t *pcm, uint32_t U, uint32_t B, uint32_t n_len,
                                      const sr_recog_out *o) {
    return recognise_dev_impl(h, pcm, U, B, n_len, o, false);
}

// sr_recog_out field by field: f(member, the handle's device mirror of it, bytes per utterance); score holds one word per
// template of the handle's bank
template <class F> static void for_each_output(sr_handle *h, F f) {
    f(&sr_recog_out::atap, h->atap, sizeof(atap_tag));
    f(&sr_recog_out::seg_off, h->seg, (size_t)24);
    f(&sr_recog_out::ftr, h->ftr, (size_t)kFtrBytes);
    f(&sr_recog_out::score, h->score, (size_t)h->bank.n * 4);
    f(&sr_recog_out::best_idx, h->bidx, (size_t)4);
    f(&sr_recog_out::best_dis, h->bdis, (size_t)4);
    f(&sr_recog_out::cmd, h->cmd, (size_t)4);
    f(&sr_recog_out::status, h->status, (size_t)1);
}

// the outputs of utterances [lo, ...) of o; NULL fields stay NULL
static sr_recog_out recog_slice(sr_handle *h, const sr_recog_out &o, size_t lo) {
    sr_recog_out s = o;
    for_each_output(h, [&](auto m, DevBuf &, size_t bytes) { if (s.*m) s.*m += lo * bytes / sizeof *(s.*m); });
    return s;
}

// the front end of spch_recg and save_mdl on B staged utterances: noise_atap, VAD, get_mfcc of segment 0, status
static int front_end(sr_handle *h, const u16 *pcm, u32 U, u32 B, u32 n_len, atap_tag *atap, u32 *seg, void *ftr, u8 *status) {
    // main.c:258-260 noise_atap + VAD (one fused launch on the staged utterance)
    SR_LAUNCH(h, TAG_VAD, launch_vad(pcm, U, B, n_len, U, 1, 1, atap, seg, h->num_sms, h->stream, vad_work(h)));
    // main.c:268 get_mfcc of segment 0
    SR_LAUNCH(h, TAG_MFCC, launch_mfcc_h(h, pcm, U, B, seg, 6, atap, ftr));
    SR_LAUNCH(h, TAG_STATUS, launch_status(seg, ftr, B, status, h->stream));
    return 0;
}

// wait_comm: order the template scan (the first kernel that rewrites score / best) after the handle's pending collective,
// so that an all-gather of the previous batch overlaps this batch's VAD and MFCC (sr_comm.cu)
int recognise_dev_impl(sr_handle *h, const uint16_t *pcm, uint32_t U, uint32_t B, uint32_t n_len, const sr_recog_out *o,
                       bool wait_comm) {
    SR_REQUIRE(h, h && o && (B == 0 || pcm));
    SR_REQUIRE(h, U <= 65535u && n_len <= U);
    if (B == 0) return 0;
    DeviceGuard g(h->device);
    atap_tag *atap = o->atap;
    SR_CK(h, atap_or_zeroed(h, h->atap, B, atap));
    u32 *seg = o->seg_off;
    SR_CK(h, caller_or_ws(h->seg, (size_t)B * 24, seg));
    v_ftr_tag *ftr = o->ftr;
    SR_CK(h, caller_or_ws(h->ftr, (size_t)B * kFtrBytes, ftr));
    u8 *status = o->status;
    SR_CK(h, caller_or_ws(h->status, (size_t)B, status));
    if (const int rc = front_end(h, pcm, U, B, n_len, atap, seg, ftr, status)) return rc;
    if (h->comm) {                                       // collectives of earlier calls may still read score / the key buffer
        const int rc = wait_comm ? comm_wait_before_scan(h, o->score) : sr_comm_wait(h);
        if (rc) return rc;
    }
    // main.c:276-294 template scan (the handle's matcher, save_sign honoured as main.c:283 does), argmin, command index
    return dtw_dev_impl(h, h->bank, ftr, B, SR_DTW_CHECK_SIGN | h->match_flags, h->match_r, o->score, o->best_idx,
                        o->best_dis, o->cmd, status);
}

// sr_dtw_batch of B host inputs against `bank`, inside the host call c
static int dtw_host(HostCall &c, const BankView &bank, const v_ftr_tag *in, uint32_t B, uint32_t flags, int band_r,
                    uint32_t *score, uint32_t *best_idx, uint32_t *best_dis) {
    sr_handle *h = c.h;
    const v_ftr_tag *d_in = c.in(h->ftr, in, (size_t)B * kFtrBytes);
    u32 *d_score = score ? c.out(h->score, score, (size_t)B * bank.n * 4) : nullptr;
    u32 *d_idx = c.out(h->bidx, best_idx, (size_t)B * 4), *d_dis = c.out(h->bdis, best_dis, (size_t)B * 4);
    c.run([&] { return dtw_dev_impl(h, bank, d_in, B, flags, band_r, d_score, best_idx ? d_idx : nullptr,
                                    best_dis ? d_dis : nullptr, nullptr, nullptr); });
    return c.finish();
}

// the FFT of n inputs, 1024-point packed (re | im<<16) or `len` real samples each: raw bins and / or magnitudes
static int fft_host(HostCall &c, const uint32_t *packed, const int16_t *frames, uint32_t len, uint32_t n, uint32_t *raw,
                    uint32_t *mag) {
    sr_handle *h = c.h;
    const void *d_in = packed ? (const void *)c.in(h->scratch[0], packed, (size_t)n * 4096)
                              : (const void *)c.in(h->scratch[0], frames, (size_t)n * len * 2, 16);
    u32 *d_raw = raw ? c.out(h->scratch[1], raw, (size_t)n * 4096) : nullptr;   // copied back before mag: see fft()
    u32 *d_mag = mag ? c.out(h->scratch[2], mag, (size_t)n * 2048) : nullptr;
    c.launch(TAG_NONE, "launch_fft_generic", [&] {
        return launch_fft_generic(packed ? static_cast<const u32 *>(d_in) : nullptr, packed ? nullptr : static_cast<const s16 *>(d_in),
                                  len, n, d_raw, d_mag, h->stream);
    });
    return c.finish();
}

// sr_recognise_batch on B captures of U_in samples at the rate r (host memory; checked by the caller): chunks of about
// 32 MB of input through PcmGroups and the transport, which count input bytes. At another rate each chunk, once staged
// (and expanded, when it came packed), gets one K15 launch (tag 15) into pcm8, rows of U8 = ceil(U_in * L / M) samples, and
// is recognised there. One pcm8 chunk is enough: on the handle's stream K15 of chunk c + 1 follows the recognition of c.
static int recognise_host(sr_handle *h, const char *name, const uint16_t *pcm, u32 U_in, u32 B, const ResampleRate &r,
                          u32 n_len, const sr_recog_out *o) {
    HostCall c(h, name);
    const u32 U = (u32)rate_len(U_in, r);               // the 8 kHz row
    // chunk: ~32 MB of input PCM, a multiple of 8 utterances (keeps every chunk base 16-byte aligned)
    uint32_t chunk = (uint32_t)(((size_t)32 << 20) / ((size_t)U_in * 2));
    chunk = chunk < 8 ? 8 : (chunk & ~7u);
    if (chunk > B) chunk = B;
    const PcmGroups pg(c, U_in, B, chunk);
    u16 *pcm8 = r.rate == 8000 ? nullptr : c.ws<u16>(h->pcm8, (size_t)chunk * U * 2 + 16);
    sr_recog_out d;                                     // device mirrors of the non-NULL outputs
    memset(&d, 0, sizeof d);
    for_each_output(h, [&](auto m, DevBuf &buf, size_t bytes) {
        if (!(o->*m)) return;
        // atap is in/out: noise_atap leaves it untouched when n_len % 240 != 0 (VAD.C:33-36); so is ftr: get_mfcc writes
        // frm_num and rows < frm_num only (MFCC.C), the caller's other bytes must come back as they were
        if constexpr (std::is_same_v<decltype(m), atap_tag *sr_recog_out::*> || std::is_same_v<decltype(m), v_ftr_tag *sr_recog_out::*>)
            c.in(buf, o->*m, B * bytes);
        d.*m = c.out(buf, o->*m, B * bytes);
    });
    uint32_t issued = 0;
    // one chunk: H2D (plain u16, or 12-bit packed + expansion on the device) -> K15 at a rate -> kernels on its slice of
    // the outputs. The transport sends the issued-th chunk through buffer issued & 1.
    auto step = [&](uint32_t ci, int buf, const void *packed_src) -> int {
        const uint32_t b0 = ci * chunk, nb = (b0 + chunk <= B) ? chunk : B - b0;
        const size_t ns = (size_t)nb * U_in;
        u16 *dpcm = pg.buf(buf);
        if (packed_src) SR_CK(h, pg.send(issued, h->transport.device_stage(buf), packed_src, ns / 2 * 3));
        else SR_CK(h, pg.send(issued, dpcm, pcm + (size_t)b0 * U_in, ns * 2));
        if (packed_src) SR_LAUNCH(h, TAG_NONE, launch_unpack12(h->transport.device_stage(buf), ns, dpcm, h->stream));
        const u16 *p8 = dpcm;
        if (pcm8) {
            SR_LAUNCH(h, TAG_RESAMPLE, launch_resample_adc12(dpcm, U_in, nb, nullptr, r.rate, pcm8, U, nullptr, h->device, h->stream));
            p8 = pcm8;
        }
        const sr_recog_out dc = recog_slice(h, d, b0);
        if (const int rc = sr_recognise_batch_dev(h, p8, U, nb, n_len, &dc)) return rc;
        SR_CK(h, pg.done(issued++));
        return 0;
    };
    c.run([&] { return h->transport.send(h, pcm, U_in, B, chunk, step); });
    const int rc = c.finish();
    if (rc == 0) h->transport.call_done((uint64_t)B * U_in * 2);
    return rc;
}

// save_mdl's body on B staged captures of U samples at 8 kHz (d_pcm, stage_captures): sr_enrol_batch and its form at a rate
static int enrol_host(HostCall &c, const u16 *d_pcm, u32 U, u32 B, u32 n_len, void *bank_out, u32 slot_stride, u8 *status) {
    sr_handle *h = c.h;
    atap_tag *d_atap = c.atap(h->atap, nullptr, B, false);
    u32 *d_seg = c.ws<u32>(h->seg, (size_t)B * 24);
    void *d_ftr = c.ws(h->ftr, (size_t)B * kFtrBytes);
    u8 *d_status = c.out(h->status, status, (size_t)B);
    void *d_bank = c.out(h->scratch[0], bank_out, (size_t)B * slot_stride);
    c.run([&] { return front_end(h, d_pcm, U, B, n_len, d_atap, d_seg, d_ftr, d_status); });
    c.launch(TAG_NONE, "launch_pack_slots", [&] { return launch_pack_slots(d_ftr, d_status, B, d_bank, slot_stride, h->stream); });
    return c.finish();
}

extern "C" {

// ---- host-buffer entry points ---------------------------------------------------------------------

int sr_noise_atap_batch(sr_handle *h, const uint16_t *pcm, uint32_t U, uint32_t B, uint32_t n_len, atap_tag *atap) {
    SR_REQUIRE(h, h && (B == 0 || (pcm && atap)));
    if (B == 0) return 0;
    HostCall c(h, "sr_noise_atap_batch");
    const u16 *d_pcm = c.in(h->pcm, pcm, (size_t)B * U * 2, 16);
    atap_tag *d_atap = c.atap(h->atap, atap, B, true);
    c.run([&] { return sr_noise_atap_batch_dev(h, d_pcm, U, B, n_len, d_atap); });
    return c.finish();
}

int sr_vad_batch(sr_handle *h, const uint16_t *pcm, uint32_t U, uint32_t B, uint32_t buf_len, const atap_tag *atap,
                 uint32_t *seg_off) {
    SR_REQUIRE(h, h && (B == 0 || (pcm && atap && seg_off)));
    if (B == 0) return 0;
    HostCall c(h, "sr_vad_batch");
    const u16 *d_pcm = c.in(h->pcm, pcm, (size_t)B * U * 2, 16);
    const atap_tag *d_atap = c.in(h->atap, atap, (size_t)B * sizeof(atap_tag));
    u32 *d_seg = c.out(h->seg, seg_off, (size_t)B * 24);
    c.run([&] { return sr_vad_batch_dev(h, d_pcm, U, B, buf_len, d_atap, d_seg); });
    return c.finish();
}

int sr_mfcc_batch(sr_handle *h, const uint16_t *pcm, uint32_t U, uint32_t B, const uint32_t *seg, uint32_t seg_stride,
                  const atap_tag *atap, v_ftr_tag *ftr) {
    SR_REQUIRE(h, h && (B == 0 || (pcm && seg && atap && ftr)));
    SR_REQUIRE(h, seg_stride >= 2);
    if (B == 0) return 0;
    HostCall c(h, "sr_mfcc_batch");
    const u16 *d_pcm = c.in(h->pcm, pcm, (size_t)B * U * 2, 16);
    const atap_tag *d_atap = c.in(h->atap, atap, (size_t)B * sizeof(atap_tag));
    const u32 *d_seg = c.in(h->seg, seg, (size_t)B * seg_stride * 4);
    v_ftr_tag *d_ftr = c.in(h->ftr, ftr, (size_t)B * kFtrBytes);     // in / out: rows >= frm_num keep the caller's bytes
    c.out(h->ftr, ftr, (size_t)B * kFtrBytes);
    c.run([&] { return sr_mfcc_batch_dev(h, d_pcm, U, B, d_seg, seg_stride, d_atap, d_ftr); });
    return c.finish();
}

int sr_dtw_batch(sr_handle *h, const v_ftr_tag *in, uint32_t B, uint32_t flags, int band_r, uint32_t *score,
                 uint32_t *best_idx, uint32_t *best_dis) {
    SR_REQUIRE(h, h && (B == 0 || in));
    ScanPlan p;                                                             // before any copy: nothing is written
    SR_REQUIRE(h, scan_plan(flags, band_r, B ? h->bank.n : 0, false, &p));
    if (B == 0) return 0;
    HostCall c(h, "sr_dtw_batch");
    return dtw_host(c, h->bank, in, B, flags, band_r, score, best_idx, best_dis);
}

int sr_set_transport(sr_handle *h, int mode) {
    SR_REQUIRE(h, h && mode >= -1 && mode <= 1);
    h->transport.mode = mode;
    return 0;
}

int sr_transport_stats(const sr_handle *h, uint32_t *packed_chunks, uint32_t *plain_chunks, uint64_t *h2d_bytes) {
    if (!h) return -1;
    if (packed_chunks) *packed_chunks = h->transport.last_packed;
    if (plain_chunks) *plain_chunks = h->transport.last_plain;
    if (h2d_bytes) *h2d_bytes = h->transport.last_h2d;
    return 0;
}

uint32_t sr_debug_pack12_host(int variant, const uint16_t *src, uint64_t n, uint8_t *dst) {
    if (!src || !dst || (n & 1)) return 0xFFFFFFFFu;
    if (variant >= 100) { PackPool pool(variant - 100); uint32_t o = 0; for (int rep = 0; rep < 3; ++rep) o = pool.run(src, (size_t)n, dst); return o; }   // the worker pool (3 fork-joins)
    return variant < 0 ? pack12(src, (size_t)n, dst) : pack12_variant(variant, src, (size_t)n, dst);
}

int sr_debug_unpack12(sr_handle *h, const uint8_t *packed, uint64_t n, uint16_t *out) {
    SR_REQUIRE(h, h && packed && out && !(n & 1));
    if (n == 0) return 0;
    HostCall c(h, "sr_debug_unpack12");
    const u8 *d_packed = c.in(h->scratch[0], packed, (size_t)(n / 2 * 3), 64);
    u16 *d_out = c.out(h->scratch[1], out, (size_t)n * 2, 64);
    c.launch(TAG_NONE, "launch_unpack12", [&] { return launch_unpack12(d_packed, n, d_out, h->stream); });
    return c.finish();
}

// Host-buffer spch_recg for B utterances. Large batches are processed in chunks through two device PCM
// buffers: the H2D copy of chunk c+1 (copy stream) overlaps the kernels of chunk c (compute stream), so
// with pinned host memory the call is bound by max(PCIe, compute) instead of their sum.
int sr_recognise_batch(sr_handle *h, const uint16_t *pcm, uint32_t U, uint32_t B, uint32_t n_len, const sr_recog_out *o) {
    SR_REQUIRE(h, h && o && (B == 0 || pcm));
    SR_REQUIRE(h, capture_args_ok(U, B, n_len));
    if (B == 0) return 0;
    return recognise_host(h, "sr_recognise_batch", pcm, U, B, kRate8k, n_len, o);
}

// at 8000 the 8 kHz call itself; else recognise_host's K15 on each chunk before its recognition
int sr_recognise_batch_at_rate(sr_handle *h, const uint16_t *pcm, uint32_t U_in, uint32_t B, uint32_t rate, uint32_t n_len,
                               const sr_recog_out *o) {
    SR_REQUIRE(h, h && o && (B == 0 || pcm));
    ResampleRate r;
    SR_REQUIRE(h, capture_rate_args_ok(rate, U_in, B, n_len, &r));
    if (rate == 8000) return sr_recognise_batch(h, pcm, U_in, B, n_len, o);
    if (B == 0) return 0;
    return recognise_host(h, "sr_recognise_batch_at_rate", pcm, U_in, B, r, n_len, o);
}

// save_mdl (main.c:121-138) for B utterances: noise_atap -> VAD -> get_mfcc(seg 0) -> save_ftr_mdl into slot b of a
// flash-layout bank image (host memory, B x slot_stride bytes). status[b]: 0 save_ok, 1 VAD_fail, 2 MFCC_fail
// (main.c:38-40); failed slots stay erased (0xFF). The result can be handed to sr_set_bank unchanged.
int sr_enrol_batch(sr_handle *h, const uint16_t *pcm, uint32_t U, uint32_t B, uint32_t n_len, void *bank_out,
                   uint32_t slot_stride, uint8_t *status) {
    SR_REQUIRE(h, h && (B == 0 || (pcm && bank_out)));
    SR_REQUIRE(h, capture_args_ok(U, B, n_len) && slot_stride >= (uint32_t)kFtrBytes && slot_stride % 4 == 0);
    if (B == 0) return 0;
    HostCall c(h, "sr_enrol_batch");
    return enrol_host(c, stage_captures(c, pcm, U, B, kRate8k), U, B, n_len, bank_out, slot_stride, status);
}

// at 8000 the 8 kHz call itself; else stage_captures' K15 before the 8 kHz body
int sr_enrol_batch_at_rate(sr_handle *h, const uint16_t *pcm, uint32_t U_in, uint32_t B, uint32_t rate, uint32_t n_len,
                           void *bank_out, uint32_t slot_stride, uint8_t *status) {
    SR_REQUIRE(h, h && (B == 0 || (pcm && bank_out)));
    ResampleRate r;
    SR_REQUIRE(h, capture_rate_args_ok(rate, U_in, B, n_len, &r) && slot_stride >= (uint32_t)kFtrBytes && slot_stride % 4 == 0);
    if (rate == 8000) return sr_enrol_batch(h, pcm, U_in, B, n_len, bank_out, slot_stride, status);
    if (B == 0) return 0;
    HostCall c(h, "sr_enrol_batch_at_rate");
    return enrol_host(c, stage_captures(c, pcm, U_in, B, r), (u32)rate_len(U_in, r), B, n_len, bank_out, slot_stride, status);
}

// get_mdl (DTW.C:217-296) for n pairs: mdl[p] = average of in1[p], in2[p] along their greedy DTW path; dis[p] = the
// path's step-normalised distance (dis_err and mdl[p] untouched when the 2:1 length guard rejects the pair).
int sr_get_mdl_batch(sr_handle *h, const v_ftr_tag *in1, const v_ftr_tag *in2, uint32_t n, v_ftr_tag *mdl, uint32_t *dis) {
    SR_REQUIRE(h, h && (n == 0 || (in1 && in2 && mdl)));
    if (n == 0) return 0;
    HostCall c(h, "sr_get_mdl_batch");
    const size_t bytes = (size_t)n * kFtrBytes;
    const v_ftr_tag *d_in1 = c.in(h->scratch[0], in1, bytes), *d_in2 = c.in(h->scratch[1], in2, bytes);
    v_ftr_tag *d_mdl = c.in(h->ftr, mdl, bytes);                    // rejected pairs leave mdl as the caller passed it
    c.out(h->ftr, mdl, bytes);
    u32 *d_dis = c.out(h->bdis, dis, (size_t)n * 4);
    c.launch(TAG_NONE, "launch_get_mdl", [&] { return launch_get_mdl(d_in1, d_in2, d_mdl, n, d_dis, h->stream); });
    return c.finish();
}

// The banded DP of n (in[p], mdl[p]) pairs with its optimal warping path (dtw_align_kernel): dis[p] is the score of
// sr_dtw_batch with SR_DTW_BAND, path[p] the (i, j) points from (0, 0) to (I-1, M-1), 0xFF past path_len[p].
int sr_dtw_path_batch(sr_handle *h, const v_ftr_tag *in, const v_ftr_tag *mdl, uint32_t n, int band_r, uint8_t *path,
                      uint32_t *path_len, uint32_t *dis) {
    SR_REQUIRE(h, h && (n == 0 || (in && mdl && dis)));
    SR_REQUIRE(h, band_r >= 0);
    if (n == 0) return 0;
    HostCall c(h, "sr_dtw_path_batch");
    const size_t bytes = (size_t)n * kFtrBytes;
    const v_ftr_tag *d_in = c.in(h->align.in_bank, in, bytes), *d_mdl = c.in(h->align.mdl_out, mdl, bytes);
    u8 *d_path = path ? c.out(h->align.path, path, (size_t)n * SR_PATH_MAX * 2) : nullptr;
    u32 *d_len = path_len ? c.out(h->align.len_pairs, path_len, (size_t)n * 4) : nullptr;
    u32 *d_dis = c.out(h->align.dis_tpl, dis, (size_t)n * 4);
    c.launch(TAG_ALIGN, "launch_dtw_align", [&] {
        return launch_dtw_align(d_in, kFtrBytes, d_mdl, kFtrBytes, nullptr, n, band_r, d_path, d_len, d_dis, nullptr, nullptr,
                                0, nullptr, nullptr, h->num_sms, h->stream);
    });
    return c.finish();
}

// DTW barycentre averaging of G groups of K consecutive slots of a flash-layout bank image. Membership, the pair lists and
// the per-group status come from the slot headers on the host; then every pass runs on the device, in one stream order:
// the anchor scores S(l -> k) of every member pair, per iteration an alignment of every member to the group's template
// (the first one resolves the anchor from S and copies it in as C_0) and an update, the final scores, and the packing of
// slot g*K (the template, signed) with the group's other K-1 slots erased: one pack of G slots K*slot_stride bytes wide.
int sr_average_bank(sr_handle *h, const void *bank, uint32_t slot_stride, uint32_t K, uint32_t G, int band_r, uint32_t iters,
                    void *bank_out, uint32_t *score, uint32_t *anchor) {
    SR_REQUIRE(h, h && (G == 0 || (bank && bank_out)));
    SR_REQUIRE(h, band_r >= 0 && K >= 1 && K <= 32 && slot_stride >= (uint32_t)kFtrBytes && slot_stride % 4 == 0);
    SR_REQUIRE(h, (uint64_t)K * slot_stride <= 0xFFFFFFFFull);
    if (G == 0) return 0;
    const auto *b = static_cast<const unsigned char *>(bank);
    const size_t slots = (size_t)G * K;
    std::vector<u32> mask(G, 0), pairs, mpairs;          // pairs: (input slot, template slot, S index) of the anchor pass
    std::vector<u8> gst(G, SR_ST_VAD_FAIL);              // a group without members packs as failed: all K slots erased
    for (u32 g = 0; g < G; ++g) {
        for (u32 k = 0; k < K; ++k) {
            u32 hdr;
            memcpy(&hdr, b + ((size_t)g * K + k) * slot_stride, 4);
            const u32 frm = hdr >> 16;
            if ((hdr & 0xFFFFu) == SR_SAVE_MASK && frm >= 1 && frm <= SR_VV_FRM_MAX) mask[g] |= 1u << k;   // decode_frm's rule
        }
        if (!mask[g]) continue;
        gst[g] = SR_ST_OK;
        for (u32 l = 0; l < K; ++l) {
            if (!((mask[g] >> l) & 1u)) continue;
            mpairs.insert(mpairs.end(), {g * K + l, g, g * K + l});
            for (u32 k = 0; k < K; ++k)
                if (k != l && ((mask[g] >> k) & 1u)) pairs.insert(pairs.end(), {g * K + l, g * K + k, (g * K + l) * K + k});
        }
    }
    const u32 n_anchor = (u32)(pairs.size() / 3), n_member = (u32)(mpairs.size() / 3);
    pairs.insert(pairs.end(), mpairs.begin(), mpairs.end());
    HostCall c(h, "sr_average_bank");
    const unsigned char *d_bank = c.in(h->align.in_bank, b, slots * slot_stride);
    void *d_out = c.out(h->align.mdl_out, bank_out, slots * slot_stride);
    u8 *d_path = c.ws<u8>(h->align.path, slots * SR_PATH_MAX * 2);
    const auto *d_pairs = c.in(h->align.len_pairs, pairs.data(), pairs.size() * 4, 16);
    auto *d_tpl = c.ws<unsigned char>(h->align.dis_tpl, (size_t)G * kFtrBytes);
    u32 *d_mask = c.in(h->align.mask, mask.data(), (size_t)G * 4);
    u8 *d_st = c.in(h->align.group_status, gst.data(), G);
    u32 *d_S = c.ws<u32>(h->align.anchor_S, slots * K * 4), *d_len = c.ws<u32>(h->align.slot_len, slots * 4);
    u32 *d_score = c.out(h->score, score, slots * 4), *d_anchor = c.out(h->bidx, anchor, (size_t)G * 4);
    auto fill = [&](void *p, int v, size_t bytes) { c.ck("cudaMemsetAsync", p ? cudaMemsetAsync(p, v, bytes, h->stream) : cudaSuccess); };
    fill(d_S, 0xFF, slots * K * 4);                      // non-member pairs: SR_DIS_ERR
    fill(d_len, 0, slots * 4);
    fill(d_score, 0xFF, slots * 4);
    fill(d_anchor, 0xFF, (size_t)G * 4);                 // empty groups: no anchor
    const u32 *d_mp = d_pairs + 3 * (size_t)n_anchor;
    if (n_anchor)
        c.launch(TAG_ALIGN, "launch_dtw_align (anchor scores)", [&] {
            return launch_dtw_align(d_bank, slot_stride, d_bank, slot_stride, d_pairs, n_anchor, band_r, nullptr, nullptr, d_S,
                                    nullptr, nullptr, K, nullptr, nullptr, h->num_sms, h->stream);
        });
    for (u32 t = 0; t < iters && n_member; ++t) {
        c.launch(TAG_ALIGN, "launch_dtw_align (members to the template)", [&] {
            return launch_dtw_align(d_bank, slot_stride, d_tpl, kFtrBytes, d_mp, n_member, band_r, d_path, d_len, nullptr,
                                    t == 0 ? d_S : nullptr, d_mask, K, d_tpl, d_anchor, h->num_sms, h->stream);
        });
        c.launch(TAG_AVG_UPDATE, "launch_average_update", [&] {
            return launch_average_update(d_bank, slot_stride, K, G, d_mask, d_path, d_len, d_tpl, h->stream);
        });
    }
    if (n_member)
        c.launch(TAG_ALIGN, "launch_dtw_align (final scores)", [&] {
            return launch_dtw_align(d_bank, slot_stride, d_tpl, kFtrBytes, d_mp, n_member, band_r, nullptr, nullptr, d_score,
                                    iters == 0 ? d_S : nullptr, d_mask, K, d_tpl, d_anchor, h->num_sms, h->stream);
        });
    c.launch(TAG_NONE, "launch_pack_slots", [&] { return launch_pack_slots(d_tpl, d_st, G, d_out, K * slot_stride, h->stream); });
    return c.finish();
}

}  // extern "C"

// ---- long features and connected words ----------------------------------------------------------------------------
// get_mfcc pieces of long segments: piece k of a segment of F frames is frames [119k, min(119(k+1), F)), a segment of
// its own that starts at sample start + 80*119*k of the utterance's row (so x[-1] is pinned only for a piece at sample 0)
struct LongPieces {
    u32 frame_len;                        // the handle's geometry
    u32 rows = 0;                         // long feature row of the next segment's first frame
    std::vector<u32> seg, row, dst;       // [P][2] start / end sample, [P] PCM row, [P][2] first long feature row / frames
    std::vector<atap_tag> atap;           // [P] the utterance's
    explicit LongPieces(const sr_handle *h) : frame_len(::frame_len(h)) {}
    // segment [st, en) of PCM row r of U samples: its F frames (MFCC.C:102-107 as mfcc_frames in sr_mfcc_core.cuh counts
    // them, without the vv_frm_max cap; 0 when it has none or more than cap) as pieces at rows, which advances by F
    u32 add(u32 st, u32 en, u32 U, u32 r, const atap_tag &a, u32 cap = 0xFFFFFFFFu) {
        const bool framed = st != SR_SEG_NULL && en != SR_SEG_NULL && en <= U && st <= en && en - st >= frame_len;
        u32 F = framed ? (en - st - frame_len) / SR_FRAME_MOV + 1u : 0u;
        if (F > cap) F = 0;
        for (u32 f0 = 0; f0 < F; f0 += SR_VV_FRM_MAX) {
            const u32 nf = std::min(F - f0, SR_VV_FRM_MAX), ps = st + f0 * SR_FRAME_MOV;
            seg.insert(seg.end(), {ps, ps + (nf - 1) * SR_FRAME_MOV + frame_len});
            row.push_back(r);
            dst.insert(dst.end(), {rows + f0, nf});
            atap.push_back(a);
        }
        rows += F;
        return F;
    }
    u32 size() const { return (u32)row.size(); }
};

// spch_recg's early returns on a segment ending at en with F frames (main.c:261-274)
static u8 seg_status(u32 en, u32 F) { return en == SR_SEG_NULL ? SR_ST_VAD_FAIL : F == 0 ? SR_ST_MFCC_FAIL : SR_ST_OK; }

constexpr u32 kPieceChunk = 8192;         // pieces per get_mfcc launch: 8192 x 2860 B of piece features

// the pieces through get_mfcc in the handle's geometry (tag 1), kPieceChunk at a time, their rows gathered into d_feat
static void run_pieces(HostCall &c, const u16 *d_pcm, u32 U, u32 n_rows, const LongPieces &pc, s16 *d_feat) {
    sr_handle *h = c.h;
    const u32 P = pc.size();
    for (u32 p0 = 0; p0 < P && !c.rc; p0 += kPieceChunk) {
        const u32 np = std::min(P - p0, kPieceChunk);
        const u32 *d_seg = c.in(h->pieces.seg, pc.seg.data() + 2 * (size_t)p0, (size_t)np * 8);
        const u32 *d_row = c.in(h->pieces.row, pc.row.data() + p0, (size_t)np * 4);
        const u32 *d_dst = c.in(h->pieces.dst, pc.dst.data() + 2 * (size_t)p0, (size_t)np * 8);
        const atap_tag *d_atap = c.in(h->pieces.atap, pc.atap.data() + p0, (size_t)np * sizeof(atap_tag));
        void *d_pf = c.ws(h->pieces.ftr, (size_t)np * kFtrBytes);
        c.launch(TAG_MFCC, "launch_mfcc_h (pieces)", [&] { return launch_mfcc_h(h, d_pcm, U, np, d_seg, 2, d_atap, d_pf, d_row, n_rows); });
        c.launch(TAG_NONE, "launch_conn_gather", [&] { return launch_conn_gather(d_pf, d_dst, np, d_feat, h->num_sms, h->stream); });
    }
}

// the device copies of a connected call's outputs, each NULL when the caller passes none: word records (in / out: records
// past n_words keep the caller's bytes), word counts and totals
struct ConnDev {
    sr_conn_word *words; u32 *nw; u64 *total;
    // the outputs of sequences b0, ...
    ConnDev at(u32 b0, u32 max_words) const {
        return {words ? words + (size_t)b0 * max_words : nullptr, nw ? nw + b0 : nullptr, total ? total + b0 : nullptr};
    }
};
static ConnDev conn_outputs(HostCall &c, u32 B, u32 max_words, sr_conn_word *words, u32 *n_words, uint64_t *total) {
    sr_handle *h = c.h;
    ConnDev d{nullptr, nullptr, nullptr};
    const size_t wbytes = (size_t)B * max_words * sizeof(sr_conn_word);
    if (words && max_words) {
        d.words = c.in(h->conn.words, words, wbytes);
        c.out(h->conn.words, words, wbytes);
    }
    d.nw = n_words ? c.out(h->conn.n_words, n_words, (size_t)B * 4) : nullptr;
    d.total = total ? c.out(h->conn.total, reinterpret_cast<u64 *>(total), (size_t)B * 8) : nullptr;
    return d;
}

// noise_atap + VAD of B captures of U samples from d_pcm (o->atap in / out: untouched when n_len % 240 != 0, else zeros),
// then one synchronisation: the plan needs the segments. seg [B][6] and atap [B] come back on the host.
static void conn_vad(HostCall &c, const u16 *d_pcm, u32 U, u32 B, u32 n_len, const sr_conn_out *o, std::vector<u32> &seg,
                     std::vector<atap_tag> &atap) {
    sr_handle *h = c.h;
    atap_tag *d_atap = c.atap(h->atap, o->atap, B, false);
    u32 *d_seg = c.ws<u32>(h->seg, (size_t)B * 24);
    c.launch(TAG_VAD, "launch_vad", [&] { return launch_vad(d_pcm, U, B, n_len, U, 1, 1, d_atap, d_seg, h->num_sms, h->stream, vad_work(h)); });
    seg.assign((size_t)B * 6, 0);
    atap.assign(B, atap_tag{});
    if (d_seg) c.ck("copy back", cudaMemcpyAsync(seg.data(), d_seg, (size_t)B * 24, cudaMemcpyDeviceToHost, h->stream));
    if (d_atap) c.ck("copy back", cudaMemcpyAsync(atap.data(), d_atap, (size_t)B * sizeof(atap_tag), cudaMemcpyDeviceToHost, h->stream));
    c.ck("cudaStreamSynchronize", cudaStreamSynchronize(h->stream));
}

// the end of a recognise-connected call: finish c, then the host-side outputs of the plan
static int conn_finish(HostCall &c, const sr_conn_out *o, u32 B, const std::vector<atap_tag> &atap, const std::vector<u32> &seg,
                       const std::vector<u32> &frm, const std::vector<u8> &status) {
    const int rc = c.finish();
    if (rc) return rc;
    if (o->atap) memcpy(o->atap, atap.data(), (size_t)B * sizeof(atap_tag));
    if (o->seg_off) memcpy(o->seg_off, seg.data(), (size_t)B * 24);
    if (o->frm_num) memcpy(o->frm_num, frm.data(), (size_t)B * 12);
    if (o->status) memcpy(o->status, status.data(), B);
    return 0;
}

// noise_atap + VAD of B staged captures of U samples at 8 kHz (d_pcm, stage_captures), then (after one synchronisation:
// the piece plan needs the segments) the long features of every closed segment packed back to back, one decoder sequence
// per segment with frames, and the join of each capture's segments: sr_recognise_connected_batch and its form at a rate
static int connected_host(HostCall &c, const u16 *d_pcm, u32 U, u32 B, u32 n_len, u32 penalty, u32 max_words,
                          const sr_conn_out *o) {
    sr_handle *h = c.h;
    std::vector<u32> seg;
    std::vector<atap_tag> atap;
    conn_vad(c, d_pcm, U, B, n_len, o, seg, atap);
    if (c.rc) return c.finish();
    // the plan: sequence q = the q-th closed segment with frames; rows and word records packed at seq_off[q][0] (frames)
    std::vector<u32> frm((size_t)B * 3), seq_of((size_t)B * 3, 0xFFFFFFFFu), seq_off, seq_frm;
    std::vector<u8> status(B);
    LongPieces pc(h);
    for (u32 b = 0; b < B; ++b) {
        for (u32 k = 0; k < 3; ++k) {
            const u32 r0 = pc.rows, F = pc.add(seg[b * 6 + 2 * k], seg[b * 6 + 2 * k + 1], U, b, atap[b]);   // <= 818: U <= 65535
            frm[b * 3 + k] = F;
            if (!F) continue;
            seq_of[b * 3 + k] = (u32)seq_frm.size();
            seq_off.insert(seq_off.end(), {r0, r0});
            seq_frm.push_back(F);
        }
        status[b] = seg_status(seg[b * 6 + 1], frm[b * 3]);
    }
    const u32 nseq = (u32)seq_frm.size(), rows = pc.rows;
    s16 *d_feat = c.ws<s16>(h->conn.feat, (size_t)rows * 24);
    run_pieces(c, d_pcm, U, B, pc, d_feat);
    const u32 *d_soff = c.in(h->conn.seq_off, seq_off.data(), (size_t)nseq * 8);
    const u32 *d_sfrm = c.in(h->conn.seq_frm, seq_frm.data(), (size_t)nseq * 4);
    const u32 *d_sof = c.in(h->conn.seq_of, seq_of.data(), (size_t)B * 12);
    sr_conn_word *d_sw = c.ws<sr_conn_word>(h->conn.seq_words, (size_t)rows * sizeof(sr_conn_word));
    u64 *d_stot = c.ws<u64>(h->conn.seq_total, (size_t)nseq * 8);
    u32 *d_snw = c.ws<u32>(h->conn.seq_n_words, (size_t)nseq * 4);
    const BankView &bk = h->bank;
    for (u32 b0 = 0; b0 < nseq; b0 += kSeqChunk)
        c.launch(TAG_CONN, "launch_dtw_connected", [&] {
            return launch_dtw_connected(d_feat, 0, d_sfrm, d_soff, b0, std::min(nseq - b0, kSeqChunk), bk.p, bk.n, bk.stride,
                                        penalty, 0, d_sw, d_snw, d_stot, h->stream);
        });
    const ConnDev d = conn_outputs(c, B, max_words, o->words, o->n_words, o->total);
    if (d.words || d.nw || d.total)
        c.launch(TAG_NONE, "launch_conn_concat", [&] {
            return launch_conn_concat(d_sof, d_soff, d_sw, d_snw, d_stot, B, max_words, d.words, d.nw, d.total, h->stream);
        });
    return conn_finish(c, o, B, atap, seg, frm, status);
}

extern "C" {

// get_mfcc with vv_frm_max replaced by frm_cap: the frame counts and the piece plan come from the segment offsets on the
// host, every feature row from the get_mfcc kernel
int sr_mfcc_long_batch(sr_handle *h, const uint16_t *pcm, uint32_t U, uint32_t B, const uint32_t *seg, uint32_t seg_stride,
                       const atap_tag *atap, uint32_t frm_cap, int16_t *feat, uint32_t *frm_num) {
    SR_REQUIRE(h, h && (B == 0 || (pcm && seg && atap && feat && frm_num)));
    SR_REQUIRE(h, seg_stride >= 2 && frm_cap >= 1 && frm_cap <= SR_CONN_FRM_MAX && (uint64_t)B * frm_cap < (1ull << 32));
    if (B == 0) return 0;
    std::vector<u32> F(B);
    LongPieces pc(h);
    for (u32 b = 0; b < B; ++b) {
        pc.rows = b * frm_cap;
        F[b] = pc.add(seg[(size_t)b * seg_stride], seg[(size_t)b * seg_stride + 1], U, b, atap[b], frm_cap);
    }
    HostCall c(h, "sr_mfcc_long_batch");
    const size_t fbytes = (size_t)B * frm_cap * 24;
    const u16 *d_pcm = c.in(h->pcm, pcm, (size_t)B * U * 2, 16);
    s16 *d_feat = c.in(h->conn.feat, reinterpret_cast<const s16 *>(feat), fbytes);   // in / out: rows >= frm_num keep the caller's bytes
    c.out(h->conn.feat, feat, fbytes);
    run_pieces(c, d_pcm, U, B, pc, d_feat);
    const int rc = c.finish();
    if (rc == 0) memcpy(frm_num, F.data(), (size_t)B * 4);
    return rc;
}

// the one-pass DP of B feature sequences against the handle's bank (dtw_connected_kernel, tag 9)
int sr_connected_batch(sr_handle *h, const int16_t *feat, const uint32_t *frm_num, uint32_t frm_stride, uint32_t B,
                       uint32_t penalty, uint32_t max_words, sr_conn_word *words, uint32_t *n_words, uint64_t *total) {
    SR_REQUIRE(h, h && (B == 0 || (feat && frm_num && n_words)));
    if (B == 0) return 0;
    SR_REQUIRE(h, h->bank.n <= SR_CONN_SLOT_MAX);
    for (u32 b = 0; b < B; ++b) SR_REQUIRE(h, frm_num[b] <= SR_CONN_FRM_MAX && frm_num[b] <= frm_stride);
    HostCall c(h, "sr_connected_batch");
    const s16 *d_feat = c.in(h->conn.feat, feat, (size_t)B * frm_stride * 24);
    const u32 *d_frm = c.in(h->conn.seq_frm, frm_num, (size_t)B * 4);
    const ConnDev d = conn_outputs(c, B, max_words, words, n_words, total);
    const BankView &bk = h->bank;
    for (u32 b0 = 0; b0 < B; b0 += kSeqChunk)
        c.launch(TAG_CONN, "launch_dtw_connected", [&] {
            return launch_dtw_connected(d_feat, frm_stride, d_frm, nullptr, b0, std::min(B - b0, kSeqChunk), bk.p, bk.n, bk.stride,
                                        penalty, max_words, d.words, d.nw, d.total, h->stream);
        });
    return c.finish();
}

int sr_recognise_connected_batch(sr_handle *h, const uint16_t *pcm, uint32_t U, uint32_t B, uint32_t n_len, uint32_t penalty,
                                 uint32_t max_words, const sr_conn_out *o) {
    SR_REQUIRE(h, h && o && (B == 0 || pcm));
    SR_REQUIRE(h, capture_args_ok(U, B, n_len));
    if (B == 0) return 0;
    SR_REQUIRE(h, h->bank.n <= SR_CONN_SLOT_MAX);
    HostCall c(h, "sr_recognise_connected_batch");
    return connected_host(c, stage_captures(c, pcm, U, B, kRate8k), U, B, n_len, penalty, max_words, o);
}

// at 8000 the 8 kHz call itself; else stage_captures' K15 before the 8 kHz body
int sr_recognise_connected_batch_at_rate(sr_handle *h, const uint16_t *pcm, uint32_t U_in, uint32_t B, uint32_t rate,
                                         uint32_t n_len, uint32_t penalty, uint32_t max_words, const sr_conn_out *o) {
    SR_REQUIRE(h, h && o && (B == 0 || pcm));
    ResampleRate r;
    SR_REQUIRE(h, capture_rate_args_ok(rate, U_in, B, n_len, &r));
    if (rate == 8000) return sr_recognise_connected_batch(h, pcm, U_in, B, n_len, penalty, max_words, o);
    if (B == 0) return 0;
    SR_REQUIRE(h, h->bank.n <= SR_CONN_SLOT_MAX);
    HostCall c(h, "sr_recognise_connected_batch_at_rate");
    return connected_host(c, stage_captures(c, pcm, U_in, B, r), (u32)rate_len(U_in, r), B, n_len, penalty, max_words, o);
}

}  // extern "C"

// ---- connected words under a grammar ------------------------------------------------------------------------------
// g's copies against the handle's bank (sr_grammar in speech_recog.h): copy[c] = slot | state << 8 | src << 16, numbered
// state-major, then by slot. Membership comes from the bank's 4-byte headers, read from the device (sr_set_bank_dev banks
// are borrowed device memory). Fails, writing nothing, on a NULL or malformed grammar or more than SR_GRAM_COPY_MAX copies.
static int gram_copies(sr_handle *h, const sr_grammar *g, std::vector<u32> &copy) {
    SR_REQUIRE(h, g != nullptr);
    SR_REQUIRE(h, g->n_states >= 1 && g->n_states <= SR_GRAM_STATE_MAX);
    SR_REQUIRE(h, g->final_mask != 0 && (g->final_mask >> g->n_states) == 0);
    SR_REQUIRE(h, g->n_arcs == 0 || g->arcs != nullptr);
    for (u32 a = 0; a < g->n_arcs; ++a) SR_REQUIRE(h, g->arcs[a].from < g->n_states && g->arcs[a].to < g->n_states);
    SR_REQUIRE(h, h->bank.n <= SR_CONN_SLOT_MAX);
    const BankView &bk = h->bank;
    std::vector<u32> hdr(bk.n);
    if (bk.n && bk.p) {
        SR_CK(h, cudaMemcpy2DAsync(hdr.data(), 4, bk.p, bk.stride, 4, bk.n, cudaMemcpyDeviceToHost, h->stream));
        SR_CK(h, cudaStreamSynchronize(h->stream));
    }
    copy.clear();
    for (u32 to = 0; to < g->n_states; ++to)
        for (u32 t = 0; t < bk.n; ++t) {
            const u32 frm = hdr[t] >> 16;
            if ((hdr[t] & 0xFFFFu) != SR_SAVE_MASK || frm < 1 || frm > SR_VV_FRM_MAX) continue;   // decode_frm's rule
            u32 src = 0;
            for (u32 a = 0; a < g->n_arcs; ++a)
                if (g->arcs[a].to == to && ((g->arcs[a].cmd_mask >> (t / SR_FTR_PER_COMM)) & 1u)) src |= 1u << g->arcs[a].from;
            if (src) copy.push_back(t | to << 8 | src << 16);
        }
    SR_REQUIRE(h, copy.size() <= SR_GRAM_COPY_MAX);
    return 0;
}

constexpr size_t kGramRecBytes = 256u << 20;   // records per launch of either grammar decoder

// The launches of a grammar decoder over B sequences: consecutive ones whose records (frames(b) x row_bytes each) fit
// kGramRecBytes, or one alone, at most kSeqChunk per launch. first_row(b) = b's first record row; rows_max: of one launch.
struct RecordCuts {
    std::vector<u32> cut{0};                            // launch boundaries
    size_t rows_max = 0;
    template <class N, class R> RecordCuts(u32 B, size_t row_bytes, N frames, R first_row) {
        size_t rows = 0;
        for (u32 b = 0; b < B; ++b) {
            const size_t n = frames(b);
            if (rows && (rows + n) * row_bytes > kGramRecBytes) { cut.push_back(b); rows = 0; }
            first_row(b) = (u32)rows;
            rows += n;
            rows_max = std::max(rows_max, rows);
        }
        cut.push_back(B);
    }
    // launch(b0, q0, nq): sequences [b0 + q0, b0 + q0 + nq), the cut's records from row 0
    template <class F> void launches(F launch) const {
        for (size_t k = 0; k + 1 < cut.size(); ++k)
            for (u32 q0 = 0, nb = cut[k + 1] - cut[k]; q0 < nb; q0 += kSeqChunk) launch(cut[k], q0, std::min(nb - q0, kSeqChunk));
    }
};

// the copy table of both grammar decoders staged in gram.copy; a grammar without copies stages one word (C = 0: no warp
// walks, every sequence decodes to 0 words)
static u32 *stage_copies(HostCall &c, const std::vector<u32> &copy) {
    static const u32 kNoCopy = 0;
    return c.in(c.h->gram.copy, copy.empty() ? &kNoCopy : copy.data(), std::max<size_t>(copy.size(), 1) * 4);
}

// the grammar decoder (tag 10) over B sequences of frames N[b]: seq [B][3] holds each first feature row and its segments
// (the record rows are filled in here), records cut by RecordCuts.
static void run_grammar(HostCall &c, const s16 *d_feat, const std::vector<u32> &N, std::vector<u32> &seq,
                        const std::vector<u32> &copy, const sr_grammar *g, u32 penalty, u32 max_words, const ConnDev &d) {
    sr_handle *h = c.h;
    const u32 B = (u32)N.size(), S = g->n_states;
    const RecordCuts cuts(B, (size_t)S * 8, [&](u32 b) { return N[b]; }, [&](u32 b) -> u32 & { return seq[3 * (size_t)b + 1]; });
    u32 *d_copy = stage_copies(c, copy);
    u32 *d_seq = c.in(h->gram.seq, seq.data(), (size_t)B * 12);
    u32 *d_frm = c.in(h->gram.frm, N.data(), (size_t)B * 4);
    u64 *d_rec = c.ws<u64>(h->gram.rec, std::max<size_t>(cuts.rows_max, 1) * S * 8);
    const BankView &bk = h->bank;
    cuts.launches([&](u32 b0, u32 q0, u32 nq) {
        const ConnDev o = d.at(b0, max_words);
        c.launch(TAG_GRAM, "launch_dtw_grammar", [&] {
            return launch_dtw_grammar(d_feat, d_frm + b0, d_seq + 3 * (size_t)b0, q0, nq, bk.p, bk.stride, d_copy, (u32)copy.size(),
                                      S, g->final_mask, penalty, max_words, o.words, o.nw, o.total, d_rec, h->stream);
        });
    });
}

// noise_atap + VAD of B staged captures of U samples at 8 kHz (d_pcm, stage_captures), one synchronisation, the long
// features of every closed segment packed back to back (a capture's segments adjacent), then one decoder sequence per
// capture under g's copy table whose words go straight to the caller's records: sr_recognise_connected_grammar_batch and
// its form at a rate
static int connected_grammar_host(HostCall &c, const u16 *d_pcm, u32 U, u32 B, u32 n_len, const std::vector<u32> &copy,
                                  const sr_grammar *g, u32 penalty, u32 max_words, const sr_conn_out *o) {
    sr_handle *h = c.h;
    std::vector<u32> seg;
    std::vector<atap_tag> atap;
    conn_vad(c, d_pcm, U, B, n_len, o, seg, atap);
    if (c.rc) return c.finish();
    // the plan: capture b is sequence b, its segments with frames back to back from row seq[b][0]; segment k's first
    // frame in that sequence (1023: no frames) is field k of seq[b][2]
    std::vector<u32> frm((size_t)B * 3), N(B), seq((size_t)B * 3);
    std::vector<u8> status(B);
    LongPieces pc(h);
    for (u32 b = 0; b < B; ++b) {
        seq[3 * (size_t)b] = pc.rows;
        u32 segs = 0;
        for (u32 k = 0; k < 3; ++k) {
            const u32 F = pc.add(seg[b * 6 + 2 * k], seg[b * 6 + 2 * k + 1], U, b, atap[b]);
            frm[b * 3 + k] = F;
            segs |= (F ? N[b] : 1023u) << (10 * k);
            N[b] += F;
        }
        seq[3 * (size_t)b + 2] = segs;
        // VAD's segments are disjoint, so a capture of U <= 65 535 samples has at most 818 frames over its segments
        if (N[b] > SR_CONN_FRM_MAX) c.took(fail(h, "a capture's segments exceed SR_CONN_FRM_MAX frames", cudaSuccess));
        status[b] = seg_status(seg[b * 6 + 1], frm[b * 3]);
    }
    if (c.rc) return c.finish();
    s16 *d_feat = c.ws<s16>(h->conn.feat, std::max<size_t>(pc.rows, 1) * 24);
    run_pieces(c, d_pcm, U, B, pc, d_feat);
    const ConnDev d = conn_outputs(c, B, max_words, o->words, o->n_words, o->total);
    if (d.words || d.nw || d.total) run_grammar(c, d_feat, N, seq, copy, g, penalty, max_words, d);
    return conn_finish(c, o, B, atap, seg, frm, status);
}

extern "C" {

// sr_connected_batch under a grammar: the copies from the bank's headers, then the decoder (dtw_grammar_kernel, tag 10)
int sr_connected_grammar_batch(sr_handle *h, const int16_t *feat, const uint32_t *frm_num, uint32_t frm_stride, uint32_t B,
                               const sr_grammar *g, uint32_t penalty, uint32_t max_words, sr_conn_word *words, uint32_t *n_words,
                               uint64_t *total) {
    SR_REQUIRE(h, h && (B == 0 || (feat && frm_num && n_words)));
    if (B == 0) return 0;
    SR_REQUIRE(h, (uint64_t)B * frm_stride < (1ull << 32));
    for (u32 b = 0; b < B; ++b) SR_REQUIRE(h, frm_num[b] <= SR_CONN_FRM_MAX && frm_num[b] <= frm_stride);
    DeviceGuard dg(h->device);
    std::vector<u32> copy;
    if (const int rc = gram_copies(h, g, copy)) return rc;
    std::vector<u32> N(frm_num, frm_num + B), seq((size_t)B * 3);
    for (u32 b = 0; b < B; ++b) {                          // one segment at frame 0
        seq[3 * (size_t)b] = b * frm_stride;
        seq[3 * (size_t)b + 2] = 1023u << 10 | 1023u << 20;
    }
    HostCall c(h, "sr_connected_grammar_batch");
    const s16 *d_feat = c.in(h->conn.feat, feat, (size_t)B * frm_stride * 24);
    const ConnDev d = conn_outputs(c, B, max_words, words, n_words, total);
    run_grammar(c, d_feat, N, seq, copy, g, penalty, max_words, d);
    return c.finish();
}

int sr_recognise_connected_grammar_batch(sr_handle *h, const uint16_t *pcm, uint32_t U, uint32_t B, uint32_t n_len,
                                         const sr_grammar *g, uint32_t penalty, uint32_t max_words, const sr_conn_out *o) {
    SR_REQUIRE(h, h && o && (B == 0 || pcm));
    SR_REQUIRE(h, capture_args_ok(U, B, n_len));
    if (B == 0) return 0;
    DeviceGuard dg(h->device);
    std::vector<u32> copy;
    if (const int rc = gram_copies(h, g, copy)) return rc;
    HostCall c(h, "sr_recognise_connected_grammar_batch");
    return connected_grammar_host(c, stage_captures(c, pcm, U, B, kRate8k), U, B, n_len, copy, g, penalty, max_words, o);
}

// at 8000 the 8 kHz call itself; else stage_captures' K15 before the 8 kHz body
int sr_recognise_connected_grammar_batch_at_rate(sr_handle *h, const uint16_t *pcm, uint32_t U_in, uint32_t B, uint32_t rate,
                                                 uint32_t n_len, const sr_grammar *g, uint32_t penalty, uint32_t max_words,
                                                 const sr_conn_out *o) {
    SR_REQUIRE(h, h && o && (B == 0 || pcm));
    ResampleRate r;
    SR_REQUIRE(h, capture_rate_args_ok(rate, U_in, B, n_len, &r));
    if (rate == 8000) return sr_recognise_connected_grammar_batch(h, pcm, U_in, B, n_len, g, penalty, max_words, o);
    if (B == 0) return 0;
    DeviceGuard dg(h->device);
    std::vector<u32> copy;
    if (const int rc = gram_copies(h, g, copy)) return rc;
    HostCall c(h, "sr_recognise_connected_grammar_batch_at_rate");
    return connected_grammar_host(c, stage_captures(c, pcm, U_in, B, r), (u32)rate_len(U_in, r), B, n_len, copy, g, penalty,
                                  max_words, o);
}

}  // extern "C"

// ---- long-form VAD and per-segment recognition (sr_long.h) ----------------------------------------------------------
static bool long_args_ok(u32 U, u32 B, u32 n_len, u32 max_segs) {
    return U <= SR_LONG_U_MAX && n_len <= 65535u && (uint64_t)B * max_segs < (1ull << 32);
}
// the host-buffer calls' recordings also have samples, and their lengths (host memory) lie within U
static bool long_host_args_ok(u32 U, u32 B, const u32 *lens, u32 n_len, u32 max_segs) {
    if ((B && !U) || !long_args_ok(U, B, n_len, max_segs)) return false;
    for (u32 b = 0; lens && b < B; ++b)
        if (lens[b] > U) return false;
    return true;
}

// the long-form noise_atap and VAD of B recordings at pcm (device): noise_atap and the block summaries (tag 11), the
// segment pass (tag 12)
static int vad_long_impl(sr_handle *h, const u16 *pcm, u32 U, u32 B, const u32 *lens, u32 n_len, u32 max_segs, atap_tag *atap,
                         u32 *n_segs, u32 *seg_off) {
    u32 *info;
    SR_CK(h, ensure(h->lng.info, (size_t)B * long_info_stride(U) * 4, info));
    SR_LAUNCH(h, TAG_LONG_BLOCKS, launch_long_atap(pcm, U, B, lens, n_len, atap, h->stream));
    SR_LAUNCH(h, TAG_LONG_BLOCKS, launch_long_blocks(pcm, U, B, lens, atap, info, h->num_sms, h->stream));
    SR_LAUNCH(h, TAG_LONG_SEGS, launch_long_segments(U, B, lens, atap, info, max_segs, n_segs, seg_off, h->stream));
    return 0;
}

// spch_recg's decision on the first min(n_segs[b], max_segs) segments of each of B recordings (n_segs, seg_off
// [B][max_segs][2], atap: device): the flat segment table (prefix sum, then the table), get_mfcc with a row map (tag 1),
// status (2), best-init (3), the template scan with the handle's matcher (4 or 6) and the argmin scatter into rec (5).
// Every kernel after the prefix sum reads the segment count from device memory; B * max_segs bounds the launches.
static int recognise_segs_impl(sr_handle *h, const u16 *pcm, u32 U, u32 B, u32 max_segs, const atap_tag *atap, const u32 *n_segs,
                               const u32 *seg_off, sr_long_seg *rec) {
    const u32 M = B * max_segs;
    if (M == 0) return 0;
    u32 *first, *n_flat, *seg2, *row, *slot;
    atap_tag *atap_seg;
    u8 *status;
    void *ftr;
    SR_CK(h, ensure(h->lng.first, (size_t)B * 4, first));
    SR_CK(h, ensure(h->lng.n_flat, 4, n_flat));
    SR_CK(h, ensure(h->lng.seg2, (size_t)M * 8, seg2));
    SR_CK(h, ensure(h->lng.row, (size_t)M * 4, row));
    SR_CK(h, ensure(h->lng.slot, (size_t)M * 4, slot));
    SR_CK(h, ensure(h->lng.atap_seg, (size_t)M * sizeof(atap_tag), atap_seg));
    SR_CK(h, ensure(h->lng.status, (size_t)M, status));
    SR_CK(h, ensure(h->lng.ftr, (size_t)M * kFtrBytes, ftr));
    SR_LAUNCH(h, TAG_NONE, launch_long_flatten(n_segs, seg_off, atap, B, max_segs, first, n_flat, seg2, row, slot, atap_seg, h->stream, 0));
    SR_LAUNCH(h, TAG_NONE, launch_long_flatten(n_segs, seg_off, atap, B, max_segs, first, n_flat, seg2, row, slot, atap_seg, h->stream, 1));
    SR_LAUNCH(h, TAG_MFCC, launch_mfcc_h(h, pcm, U, M, seg2, 2, atap_seg, ftr, row, B, n_flat));     // main.c:268
    SR_LAUNCH(h, TAG_STATUS, launch_long_status(seg2, ftr, n_flat, M, status, h->stream));          // main.c:261-274
    // main.c:276-291, save_sign honoured (main.c:283); a decision rule's key rows in lng.keys
    ScanPlan p;
    scan_plan(SR_DTW_CHECK_SIGN | h->match_flags, h->match_r, h->bank.n, true, &p);    // flags sr_set_match accepted
    u64 *keys;
    if (const int rc = scan_to_keys(h, &h->lng.keys, p, h->bank, ftr, M, nullptr, status, keys, n_flat)) return rc;
    SR_LAUNCH(h, TAG_BEST_FINAL, launch_long_scatter(seg2, slot, ftr, status, keys, n_flat, M, rec, p.rule, h->stream));   // main.c:292-294
    return 0;
}

constexpr size_t kLongGroupBytes = (size_t)256 << 20;   // PCM per staged group of the host calls

// recordings per staged group: as many rows of U samples as fit kLongGroupBytes, at least one, at most B
static u32 long_group_size(u32 U, u32 B) { return std::max(1u, std::min((u32)(kLongGroupBytes / ((size_t)U * 2)), B)); }

// The host-buffer long-form calls: whole recordings staged in groups of G (long_group_size: at most kLongGroupBytes of
// PCM, at least one recording) through PcmGroups, and run(device PCM, first recording, recordings) per group. A recording
// is never split.
template <class F> static int long_groups(HostCall &c, const uint16_t *pcm, u32 U, u32 B, u32 G, F run) {
    const PcmGroups pg(c, U, B, G);
    for (u32 g = 0; g < pg.n && !c.rc; ++g) {
        const u32 b0 = g * pg.G, nb = std::min(pg.G, B - b0);
        u16 *dpcm = pg.buf(g & 1);
        c.ck("PcmGroups::send", pg.send(g, dpcm, pcm + (size_t)b0 * U, (size_t)nb * U * 2));
        c.run([&] { return run(static_cast<const u16 *>(dpcm), b0, nb); });
        c.ck("PcmGroups::done", pg.done(g));
    }
    return c.finish();
}

// The 8 kHz recordings the per-group body of a host-buffer long-form call runs on. The caller's rows of U_in samples
// (lens: host, or NULL) are staged by long_groups in groups of G recordings, at most kLongGroupBytes of input each, the
// caller's lens in lng.lens. At 8 kHz the body takes each staged group as it is. At another rate, group() first runs K15
// (tag 15) from the staged group into pcm8, rows of U8 = ceil(U_in * L / M) samples, and its 8 kHz lengths into
// lng.lens8, and the body takes those.
struct LongSource {
    HostCall &c;
    u32 U_in, U8, G;
    uint32_t rate;
    const u32 *d_lens = nullptr;        // the caller's lens, staged (NULL: U_in)
    u16 *pcm8 = nullptr;                // at a rate: [G][U8], G recordings per staged group
    u32 *lens8 = nullptr;               // at a rate: [B]
    LongSource(HostCall &cc, u32 U, u32 B, const u32 *lens, const ResampleRate &r)
        : c(cc), U_in(U), U8(rate_len(U, r)), G(long_group_size(U, B)), rate(r.rate) {
        d_lens = lens ? c.in(c.h->lng.lens, lens, (size_t)B * 4) : nullptr;
        if (rate == 8000) return;
        pcm8 = c.ws<u16>(c.h->pcm8, (size_t)G * U8 * 2);
        lens8 = c.ws<u32>(c.h->lng.lens8, (size_t)B * 4);
    }
    // recordings [b0, b0 + nb) staged at dpcm (rows of U_in samples) as the body reads them: pcm, row length U8, lens
    int group(const u16 *dpcm, u32 b0, u32 nb, const u16 *&pcm, const u32 *&lens) const {
        if (rate == 8000) {
            pcm = dpcm;
            lens = d_lens ? d_lens + b0 : nullptr;
            return 0;
        }
        // grid: a group holds at most 2^27 rows, or rows of 2^27 samples together, and a tile at least 2 048 outputs
        sr_handle *h = c.h;
        SR_LAUNCH(h, TAG_RESAMPLE, launch_resample_adc12(dpcm, U_in, nb, d_lens ? d_lens + b0 : nullptr, rate, pcm8, U8,
                                                         lens8 + b0, h->device, h->stream));
        pcm = pcm8;
        lens = lens8 + b0;
        return 0;
    }
};

// the argument rules of a host-buffer long-form call at a rate: the rate, U_in within K15's limit, and the 8 kHz call's
// rules on U8 (lens8 <= U8 follows from lens <= U_in)
static bool long_rate_args_ok(uint32_t rate, u32 U_in, u32 B, const u32 *lens, u32 n_len, u32 max_segs, ResampleRate *r) {
    if (!resample_rate(rate, r) || U_in > SR_RESAMPLE_U_MAX) return false;
    const uint64_t U8 = rate_len(U_in, *r);
    if (U8 > SR_LONG_U_MAX || !long_host_args_ok((u32)U8, B, nullptr, n_len, max_segs)) return false;
    for (u32 b = 0; lens && b < B; ++b)
        if (lens[b] > U_in) return false;
    return true;
}

// sr_recognise_long_batch on the recordings of src, per staged group
static int recognise_long_host(HostCall &c, const uint16_t *pcm, u32 B, const LongSource &src, u32 n_len, u32 max_segs,
                               const sr_long_out *o) {
    sr_handle *h = c.h;
    atap_tag *d_atap = c.atap(h->lng.atap, o->atap, B, true);
    u32 *d_n = o->n_segs ? c.out(h->lng.n_segs, o->n_segs, (size_t)B * 4) : nullptr;
    const size_t rbytes = (size_t)B * max_segs * sizeof(sr_long_seg);
    sr_long_seg *d_rec = nullptr;
    if (rbytes) {                                                           // in / out: records past n_segs keep the caller's bytes
        d_rec = c.in(h->lng.per_seg, o->segs, rbytes);
        c.out(h->lng.per_seg, o->segs, rbytes);
    }
    return long_groups(c, pcm, src.U_in, B, src.G, [&](const u16 *dpcm, u32 b0, u32 nb) {
        const u16 *p8;
        const u32 *l8;
        if (const int rc = src.group(dpcm, b0, nb, p8, l8)) return rc;
        const sr_long_out od{d_atap + b0, d_n ? d_n + b0 : nullptr, d_rec ? d_rec + (size_t)b0 * max_segs : nullptr};
        return sr_recognise_long_batch_dev(h, p8, src.U8, nb, l8, n_len, max_segs, &od);
    });
}

extern "C" {

int sr_vad_long_batch_dev(sr_handle *h, const uint16_t *pcm, uint32_t U, uint32_t B, const uint32_t *lens, uint32_t n_len,
                          uint32_t max_segs, atap_tag *atap, uint32_t *n_segs, uint32_t *seg_off) {
    SR_REQUIRE(h, h && (B == 0 || (pcm && atap && n_segs && (seg_off || max_segs == 0))));
    SR_REQUIRE(h, long_args_ok(U, B, n_len, max_segs));
    if (B == 0) return 0;
    DeviceGuard g(h->device);
    return vad_long_impl(h, pcm, U, B, lens, n_len, max_segs, atap, n_segs, seg_off);
}

int sr_recognise_long_batch_dev(sr_handle *h, const uint16_t *pcm, uint32_t U, uint32_t B, const uint32_t *lens, uint32_t n_len,
                                uint32_t max_segs, const sr_long_out *o) {
    SR_REQUIRE(h, h && o && (B == 0 || (pcm && (o->segs || max_segs == 0))));
    SR_REQUIRE(h, long_args_ok(U, B, n_len, max_segs));
    if (B == 0) return 0;
    DeviceGuard g(h->device);
    atap_tag *atap = o->atap;
    SR_CK(h, atap_or_zeroed(h, h->lng.atap, B, atap));
    u32 *n_segs = o->n_segs;
    SR_CK(h, caller_or_ws(h->lng.n_segs, (size_t)B * 4, n_segs));
    u32 *seg_off;
    SR_CK(h, ensure(h->lng.seg_off, (size_t)B * max_segs * 8 + 8, seg_off));
    if (const int rc = vad_long_impl(h, pcm, U, B, lens, n_len, max_segs, atap, n_segs, seg_off)) return rc;
    return recognise_segs_impl(h, pcm, U, B, max_segs, atap, n_segs, seg_off, o->segs);
}

int sr_vad_long_batch(sr_handle *h, const uint16_t *pcm, uint32_t U, uint32_t B, const uint32_t *lens, uint32_t n_len,
                      uint32_t max_segs, atap_tag *atap, uint32_t *n_segs, uint32_t *seg_off) {
    SR_REQUIRE(h, h && (B == 0 || (pcm && atap && n_segs && (seg_off || max_segs == 0))));
    SR_REQUIRE(h, long_host_args_ok(U, B, lens, n_len, max_segs));
    if (B == 0) return 0;
    HostCall c(h, "sr_vad_long_batch");
    const u32 *d_lens = lens ? c.in(h->lng.lens, lens, (size_t)B * 4) : nullptr;
    atap_tag *d_atap = c.atap(h->lng.atap, atap, B, true);
    u32 *d_n = c.out(h->lng.n_segs, n_segs, (size_t)B * 4);
    const size_t sbytes = (size_t)B * max_segs * 8;
    u32 *d_seg = nullptr;
    if (sbytes) {                                                           // in / out: segments past n_segs keep the caller's bytes
        d_seg = c.in(h->lng.per_seg, seg_off, sbytes);
        c.out(h->lng.per_seg, seg_off, sbytes);
    }
    return long_groups(c, pcm, U, B, long_group_size(U, B), [&](const u16 *dpcm, u32 b0, u32 nb) {
        return sr_vad_long_batch_dev(h, dpcm, U, nb, d_lens ? d_lens + b0 : nullptr, n_len, max_segs, d_atap + b0, d_n + b0,
                                     d_seg ? d_seg + (size_t)b0 * max_segs * 2 : nullptr);
    });
}

int sr_recognise_long_batch(sr_handle *h, const uint16_t *pcm, uint32_t U, uint32_t B, const uint32_t *lens, uint32_t n_len,
                            uint32_t max_segs, const sr_long_out *o) {
    SR_REQUIRE(h, h && o && (B == 0 || (pcm && (o->segs || max_segs == 0))));
    SR_REQUIRE(h, long_host_args_ok(U, B, lens, n_len, max_segs));
    if (B == 0) return 0;
    HostCall c(h, "sr_recognise_long_batch");
    const LongSource src(c, U, B, lens, kRate8k);
    return recognise_long_host(c, pcm, B, src, n_len, max_segs, o);
}

// at 8000 the 8 kHz call itself; else LongSource's K15 before each group's body
int sr_recognise_long_batch_at_rate(sr_handle *h, const uint16_t *pcm, uint32_t U_in, uint32_t B, const uint32_t *lens,
                                    uint32_t rate, uint32_t n_len, uint32_t max_segs, const sr_long_out *o) {
    SR_REQUIRE(h, h && o && (B == 0 || (pcm && (o->segs || max_segs == 0))));
    ResampleRate r;
    SR_REQUIRE(h, long_rate_args_ok(rate, U_in, B, lens, n_len, max_segs, &r));
    if (rate == 8000) return sr_recognise_long_batch(h, pcm, U_in, B, lens, n_len, max_segs, o);
    if (B == 0) return 0;
    HostCall c(h, "sr_recognise_long_batch_at_rate");
    const LongSource src(c, U_in, B, lens, r);
    return recognise_long_host(c, pcm, B, src, n_len, max_segs, o);
}

}  // extern "C"

// ---- one grammar decode per long recording (sr_long_grammar.h) --------------------------------------------------------
// the long-recording grammar decoder (tag 13) over the sequences of seq [B][4] (first segment, segments, frames; the first
// record row is filled in here) and the flat segment table at d_row / d_frm, records cut by RecordCuts: the record
// workspaces grow to fit a sequence whose records alone exceed the budget.
static void run_long_grammar(HostCall &c, const s16 *d_feat, std::vector<u32> &seq, const u32 *d_row, const u32 *d_frm,
                             const std::vector<u32> &copy, const sr_grammar *g, u32 penalty, u32 max_words, const ConnDev &d) {
    sr_handle *h = c.h;
    const u32 B = (u32)(seq.size() / 4), S = g->n_states;
    const RecordCuts cuts(B, (size_t)S * 12, [&](u32 b) { return seq[4 * (size_t)b + 2]; },
                        [&](u32 b) -> u32 & { return seq[4 * (size_t)b + 3]; });
    u32 *d_copy = stage_copies(c, copy);
    u32 *d_seq = c.in(h->gram.seq, seq.data(), (size_t)B * 16);
    u64 *recD = c.ws<u64>(h->gram.rec, std::max<size_t>(cuts.rows_max, 1) * S * 8);
    u32 *recS = c.ws<u32>(h->gram.rec_state, std::max<size_t>(cuts.rows_max, 1) * S * 4);
    const BankView &bk = h->bank;
    cuts.launches([&](u32 b0, u32 q0, u32 nq) {
        const ConnDev o = d.at(b0, max_words);
        c.launch(TAG_LONG_GRAM, "launch_dtw_long_grammar", [&] {
            return launch_dtw_long_grammar(d_feat, d_seq + 4 * (size_t)b0, q0, nq, d_row, d_frm, bk.p, bk.stride, d_copy,
                                           (u32)copy.size(), S, g->final_mask, penalty, max_words, o.words, o.nw, o.total, recD,
                                           recS, h->stream);
        });
    });
}

// the segment slots the end-to-end call gives the VAD per recording: a closed segment spans at least 8 + 11 = 19 VAD
// frames (8 active ones open it, 11 inactive ones close it, and the next needs 8 new active ones) and an open one at least
// 8, so a recording of U samples, with ceil((U - 160) / 80) frames, has at most frames / 19 + 1 segments
static u32 long_seg_bound(u32 U) {
    const u32 nfr = U > SR_FRAME_LEN ? (U - SR_FRAME_LEN + SR_FRAME_MOV - 1) / SR_FRAME_MOV : 0u;
    return nfr / 19u + 2u;
}

extern "C" {

// the kernel-level form: the flat segment table's rows, then the decoder (tag 13)
int sr_connected_grammar_segs_batch(sr_handle *h, const int16_t *feat, const uint32_t *seq_seg, const uint32_t *seg_frm, uint32_t B,
                                    const sr_grammar *g, uint32_t penalty, uint32_t max_words, sr_conn_word *words,
                                    uint32_t *n_words, uint64_t *total) {
    SR_REQUIRE(h, h && (B == 0 || (seq_seg && n_words)));
    if (B == 0) return 0;
    for (u32 b = 0; b < B; ++b) SR_REQUIRE(h, seq_seg[b] <= seq_seg[b + 1]);
    const u32 n_seg = seq_seg[B];
    SR_REQUIRE(h, n_seg == 0 || seg_frm);
    std::vector<u32> row(n_seg);
    uint64_t rows = 0;
    for (u32 k = 0; k < n_seg; ++k) {
        SR_REQUIRE(h, seg_frm[k] <= SR_CONN_FRM_MAX);
        row[k] = (u32)rows;
        rows += seg_frm[k];
    }
    SR_REQUIRE(h, rows < (1ull << 32) && (rows == 0 || feat));
    std::vector<u32> seq((size_t)B * 4);
    for (u32 b = 0; b < B; ++b) {
        uint64_t N = 0;
        for (u32 k = seq_seg[b]; k < seq_seg[b + 1]; ++k) N += seg_frm[k];
        SR_REQUIRE(h, N <= SR_LONG_GRAM_FRM_MAX);
        seq[4 * (size_t)b] = seq_seg[b];
        seq[4 * (size_t)b + 1] = seq_seg[b + 1] - seq_seg[b];
        seq[4 * (size_t)b + 2] = (u32)N;
    }
    DeviceGuard dg(h->device);
    std::vector<u32> copy;
    if (const int rc = gram_copies(h, g, copy)) return rc;
    HostCall c(h, "sr_connected_grammar_segs_batch");
    const s16 *d_feat = c.in(h->conn.feat, feat, (size_t)rows * 24, 24);
    u32 *d_row = c.ws<u32>(h->gram.seg_row, std::max<size_t>(n_seg, 1) * 4);
    u32 *d_frm = c.ws<u32>(h->gram.frm, std::max<size_t>(n_seg, 1) * 4);
    c.h2d(d_row, row.data(), (size_t)n_seg * 4);
    c.h2d(d_frm, seg_frm, (size_t)n_seg * 4);
    const ConnDev d = conn_outputs(c, B, max_words, words, n_words, total);
    run_long_grammar(c, d_feat, seq, d_row, d_frm, copy, g, penalty, max_words, d);
    return c.finish();
}

}  // extern "C"

// sr_recognise_long_grammar_batch on the recordings of src under the copy table of gram_copies. Per group of recordings
// (long_groups, then LongSource::group): the long-form VAD into long_seg_bound(U8) slots per recording (tags 11, 12), one
// synchronisation for the plan, the feature pieces of every decodable segment (tag 1) and one decoder sequence per
// recording over all its segments (tag 13). The per-segment records are written on the host from the plan.
static int recognise_long_grammar_host(HostCall &c, const uint16_t *pcm, u32 B, const LongSource &src,
                                       const std::vector<u32> &copy, u32 n_len, const sr_grammar *g, u32 penalty,
                                       u32 max_segs, u32 max_words, const sr_long_gram_out *o) {
    sr_handle *h = c.h;
    const u32 U = src.U8, cap = long_seg_bound(U);
    atap_tag *d_atap = c.atap(h->lng.atap, o->atap, B, true);
    u32 *d_n = c.ws<u32>(h->lng.n_segs, (size_t)B * 4);
    const ConnDev d = conn_outputs(c, B, max_words, o->words, o->n_words, o->total);
    struct SegRec { u32 b, k, st, en, F; u8 status; };    // the records of segments k < max_segs
    std::vector<SegRec> recs;
    std::vector<u32> n_all(B), segv;
    std::vector<atap_tag> av;
    const int rc = long_groups(c, pcm, src.U_in, B, src.G, [&](const u16 *dpcm_in, u32 b0, u32 nb) -> int {
        u32 *d_seg = c.ws<u32>(h->gram.vad_segs, (size_t)nb * cap * 8);
        if (c.rc) return 0;
        const u16 *dpcm;
        const u32 *d_lens;
        if (const int r = src.group(dpcm_in, b0, nb, dpcm, d_lens)) return r;
        if (const int r = vad_long_impl(h, dpcm, U, nb, d_lens, n_len, cap, d_atap + b0, d_n + b0, d_seg))
            return r;
        segv.resize((size_t)nb * cap * 2);
        av.resize(nb);
        c.ck("copy back", cudaMemcpyAsync(n_all.data() + b0, d_n + b0, (size_t)nb * 4, cudaMemcpyDeviceToHost, h->stream));
        c.ck("copy back", cudaMemcpyAsync(segv.data(), d_seg, segv.size() * 4, cudaMemcpyDeviceToHost, h->stream));
        c.ck("copy back", cudaMemcpyAsync(av.data(), d_atap + b0, (size_t)nb * sizeof(atap_tag), cudaMemcpyDeviceToHost, h->stream));
        c.ck("cudaStreamSynchronize", cudaStreamSynchronize(h->stream));
        if (c.rc) return 0;
        // the plan: recording q is sequence q; its segments are consecutive entries of the flat table, a decodable one with
        // its frames (rows packed back to back in segment order), any other with 0 frames
        std::vector<u32> seq((size_t)nb * 4), row, frm;
        LongPieces pc(h);
        for (u32 q = 0; q < nb; ++q) {
            const u32 b = b0 + q, n = n_all[b];
            if (n > cap) return fail(h, "a recording has more segments than long_seg_bound", cudaSuccess);
            seq[4 * (size_t)q] = (u32)row.size();
            seq[4 * (size_t)q + 1] = n;
            u32 N = 0;
            for (u32 k = 0; k < n; ++k) {
                const u32 st = segv[((size_t)q * cap + k) * 2], en = segv[((size_t)q * cap + k) * 2 + 1];
                row.push_back(pc.rows);
                const u32 F = pc.add(st, en, U, q, av[q], SR_CONN_FRM_MAX);   // 0 for an open segment
                frm.push_back(F);
                N += F;
                if (k < max_segs) recs.push_back({b, k, st, en, F, seg_status(en, F)});
            }
            seq[4 * (size_t)q + 2] = N;
        }
        const u32 ns = (u32)row.size();
        s16 *d_feat = c.ws<s16>(h->conn.feat, std::max<size_t>(pc.rows, 1) * 24);
        run_pieces(c, dpcm, U, nb, pc, d_feat);
        u32 *d_row = c.ws<u32>(h->gram.seg_row, std::max<size_t>(ns, 1) * 4);
        u32 *d_frm = c.ws<u32>(h->gram.frm, std::max<size_t>(ns, 1) * 4);
        c.h2d(d_row, row.data(), (size_t)ns * 4);
        c.h2d(d_frm, frm.data(), (size_t)ns * 4);
        run_long_grammar(c, d_feat, seq, d_row, d_frm, copy, g, penalty, max_words, d.at(b0, max_words));
        return 0;
    });
    if (rc) return rc;
    if (o->n_segs) memcpy(o->n_segs, n_all.data(), (size_t)B * 4);
    for (const SegRec &r : recs) {
        const size_t i = (size_t)r.b * max_segs + r.k;
        if (o->seg_off) { o->seg_off[2 * i] = r.st; o->seg_off[2 * i + 1] = r.en; }
        if (o->frm_num) o->frm_num[i] = r.F;
        if (o->seg_status) o->seg_status[i] = r.status;
    }
    return 0;
}

// One host call, several GPUs: the batch is cut into contiguous shards (SURVEY 8e), shard g runs on handles[g]
// from its own host thread, and every shard writes its results straight into its slice of the caller's host
// arrays -- with host outputs the "gather" is the D2H copies themselves, no collective is needed. (Device-resident
// multi-GPU use is one process per GPU with a NCCL all-gather of the score blocks, see bench.py.)
// All handles must have the same template bank set and the same matcher. Returns the first non-zero shard status.
// Shards of captures at 8000 Hz run sr_recognise_batch; at another rate sr_recognise_batch_at_rate, whose argument rules
// every shard applies before any copy (sr_recognise_batch_multi and its form at a rate).
static int recognise_multi(sr_handle *const *handles, uint32_t n_handles, const uint16_t *pcm, uint32_t U_in, uint32_t B,
                           uint32_t rate, uint32_t n_len, const sr_recog_out *o, const char *name) {
    const std::string nm(name);
    if (!handles || n_handles == 0 || !o) return fail(nullptr, (nm + ": bad arguments").c_str(), cudaSuccess);
    for (uint32_t g = 0; g < n_handles; ++g)
        if (!handles[g] || handles[g]->bank.n != handles[0]->bank.n) return fail(nullptr, (nm + ": handles differ").c_str(), cudaSuccess);
    for (uint32_t g = 0; g < n_handles; ++g)
        if (!same_match(handles[g], handles[0])) return fail(nullptr, (nm + ": handles differ in their matcher").c_str(), cudaSuccess);
    std::vector<int> rc(n_handles, 0);
    std::vector<std::thread> th;
    for (uint32_t g = 0; g < n_handles; ++g) {
        const uint32_t lo = (uint32_t)((uint64_t)B * g / n_handles), hi = (uint32_t)((uint64_t)B * (g + 1) / n_handles);
        const sr_recog_out s = recog_slice(handles[0], *o, lo);
        th.emplace_back([=, &rc]() {
            rc[g] = rate == 8000 ? sr_recognise_batch(handles[g], pcm + (size_t)lo * U_in, U_in, hi - lo, n_len, &s)
                                 : sr_recognise_batch_at_rate(handles[g], pcm + (size_t)lo * U_in, U_in, hi - lo, rate, n_len, &s);
        });
    }
    for (auto &t : th) t.join();
    for (uint32_t g = 0; g < n_handles; ++g) if (rc[g]) return rc[g];
    return 0;
}

extern "C" {

int sr_recognise_long_grammar_batch(sr_handle *h, const uint16_t *pcm, uint32_t U, uint32_t B, const uint32_t *lens,
                                    uint32_t n_len, const sr_grammar *g, uint32_t penalty, uint32_t max_segs, uint32_t max_words,
                                    const sr_long_gram_out *o) {
    SR_REQUIRE(h, h && o && (B == 0 || pcm));
    SR_REQUIRE(h, long_host_args_ok(U, B, lens, n_len, max_segs));
    if (B == 0) return 0;
    DeviceGuard dg(h->device);
    std::vector<u32> copy;
    if (const int rc = gram_copies(h, g, copy)) return rc;
    HostCall c(h, "sr_recognise_long_grammar_batch");
    const LongSource src(c, U, B, lens, kRate8k);
    return recognise_long_grammar_host(c, pcm, B, src, copy, n_len, g, penalty, max_segs, max_words, o);
}

// at 8000 the 8 kHz call itself; else LongSource's K15 before each group's body
int sr_recognise_long_grammar_batch_at_rate(sr_handle *h, const uint16_t *pcm, uint32_t U_in, uint32_t B, const uint32_t *lens,
                                            uint32_t rate, uint32_t n_len, const sr_grammar *g, uint32_t penalty,
                                            uint32_t max_segs, uint32_t max_words, const sr_long_gram_out *o) {
    SR_REQUIRE(h, h && o && (B == 0 || pcm));
    ResampleRate r;
    SR_REQUIRE(h, long_rate_args_ok(rate, U_in, B, lens, n_len, max_segs, &r));
    if (rate == 8000) return sr_recognise_long_grammar_batch(h, pcm, U_in, B, lens, n_len, g, penalty, max_segs, max_words, o);
    if (B == 0) return 0;
    DeviceGuard dg(h->device);
    std::vector<u32> copy;
    if (const int rc = gram_copies(h, g, copy)) return rc;
    HostCall c(h, "sr_recognise_long_grammar_batch_at_rate");
    const LongSource src(c, U_in, B, lens, r);
    return recognise_long_grammar_host(c, pcm, B, src, copy, n_len, g, penalty, max_segs, max_words, o);
}

int sr_recognise_batch_multi(sr_handle *const *handles, uint32_t n_handles, const uint16_t *pcm, uint32_t U, uint32_t B,
                             uint32_t n_len, const sr_recog_out *o) {
    return recognise_multi(handles, n_handles, pcm, U, B, 8000, n_len, o, "sr_recognise_batch_multi");
}

// at 8000 the 8 kHz call itself; else the same shards, each running sr_recognise_batch_at_rate
int sr_recognise_batch_multi_at_rate(sr_handle *const *handles, uint32_t n_handles, const uint16_t *pcm, uint32_t U_in,
                                     uint32_t B, uint32_t rate, uint32_t n_len, const sr_recog_out *o) {
    if (rate == 8000) return sr_recognise_batch_multi(handles, n_handles, pcm, U_in, B, n_len, o);
    return recognise_multi(handles, n_handles, pcm, U_in, B, rate, n_len, o, "sr_recognise_batch_multi_at_rate");
}

int sr_fft_mag_batch(sr_handle *h, const int16_t *frames, uint32_t len, uint32_t n, uint32_t *mag) {
    SR_REQUIRE(h, h && (n == 0 || (frames && mag)));
    SR_REQUIRE(h, len <= SR_FFT_POINT);                                   // MFCC.C:32-35
    if (n == 0) return 0;
    HostCall c(h, "sr_fft_mag_batch");
    return fft_host(c, nullptr, frames, len, n, nullptr, mag);
}

// dtw_limit (DTW.C:76-109) for n points, explicit (I, M) per point instead of the reference's file statics
int sr_dtw_limit_batch(sr_handle *h, const uint16_t *x, const uint16_t *y, const uint16_t *I, const uint16_t *M, uint32_t n,
                       uint8_t *out) {
    SR_REQUIRE(h, h && (n == 0 || (x && y && I && M && out)));
    if (n == 0) return 0;
    HostCall c(h, "sr_dtw_limit_batch");
    u16 *d = c.ws<u16>(h->scratch[0], (size_t)n * 8 + 16);          // x | y | I | M
    const uint16_t *src[4] = {x, y, I, M};
    for (int k = 0; k < 4; ++k) c.h2d(d + k * (size_t)n, src[k], (size_t)n * 2);
    u8 *d_out = c.out(h->scratch[2], out, (size_t)n, 16);
    c.launch(TAG_NONE, "launch_dtw_limit", [&] { return launch_dtw_limit(d, d + n, d + 2 * (size_t)n, d + 3 * (size_t)n, n, d_out, h->stream); });
    return c.finish();
}

// raw FFT of packed (re | im<<16) 1024-point inputs -- test hook for the asm restatement parity
int sr_fft_raw_batch(sr_handle *h, const uint32_t *in_packed, uint32_t n, uint32_t *out_packed) {
    SR_REQUIRE(h, h && (n == 0 || (in_packed && out_packed)));
    if (n == 0) return 0;
    HostCall c(h, "sr_fft_raw_batch");
    return fft_host(c, in_packed, nullptr, 0, n, out_packed, nullptr);
}

int sr_get_dis_batch(sr_handle *h, const int16_t *a, const int16_t *b, uint32_t n, uint32_t *dis) {
    SR_REQUIRE(h, h && (n == 0 || (a && b && dis)));
    if (n == 0) return 0;
    HostCall c(h, "sr_get_dis_batch");
    const s16 *d_a = c.in(h->scratch[0], a, (size_t)n * 24), *d_b = c.in(h->scratch[1], b, (size_t)n * 24);
    u32 *d_dis = c.out(h->scratch[2], dis, (size_t)n * 4);
    c.launch(TAG_NONE, "launch_get_dis", [&] { return launch_get_dis(d_a, d_b, n, d_dis, h->stream); });
    return c.finish();
}

// test hook: the shared MFCC core's FFT alone at N = 256 (GEOM_B) or 1024, on n packed N-point inputs
int sr_debug_fft_raw_n(sr_handle *h, const uint32_t *in_packed, uint32_t N, uint32_t n, uint32_t *out_packed) {
    SR_REQUIRE(h, h && (N == 256 || N == 1024) && (n == 0 || (in_packed && out_packed)));
    if (n == 0) return 0;
    HostCall c(h, "sr_debug_fft_raw_n");
    const u32 *d_in = c.in(h->scratch[0], in_packed, (size_t)n * N * 4);
    u32 *d_out = c.out(h->scratch[1], out_packed, (size_t)n * N * 4);
    c.launch(TAG_NONE, "launch_fft_raw_n", [&] { return launch_fft_raw_n(d_in, N, n, d_out, h->stream); });
    return c.finish();
}

// test hook: number of float bit patterns in [lo_bits, hi_bits) for which the branch-free sqrt differs from
// the IEEE intrinsic (must be 0 over [1.0f, 2^33) = the range the kernels feed it)
int sr_debug_sqrt_mismatches(sr_handle *h, uint32_t lo_bits, uint32_t hi_bits, uint64_t *mismatches) {
    SR_REQUIRE(h, h && mismatches);
    HostCall c(h, "sr_debug_sqrt_mismatches");
    auto *bad = reinterpret_cast<unsigned long long *>(c.out(h->scratch[2], mismatches, 8, 8));
    c.ck("cudaMemsetAsync", bad ? cudaMemsetAsync(bad, 0, 8, h->stream) : cudaSuccess);
    c.launch(TAG_NONE, "launch_sqrt_check", [&] { return launch_sqrt_check(lo_bits, hi_bits, bad, h->stream); });
    return c.finish();
}

// test hook: number of v in [lo, hi) for which the MFCC kernels' log100 differs from a binary search over the same
// threshold table (must be 0 over [0, 2^32))
int sr_debug_log100_mismatches(sr_handle *h, uint64_t lo, uint64_t hi, uint64_t *mismatches) {
    SR_REQUIRE(h, h && mismatches && hi <= (1ull << 32));
    HostCall c(h, "sr_debug_log100_mismatches");
    auto *bad = reinterpret_cast<unsigned long long *>(c.out(h->scratch[2], mismatches, 8, 8));
    c.ck("cudaMemsetAsync", bad ? cudaMemsetAsync(bad, 0, 8, h->stream) : cudaSuccess);
    c.launch(TAG_NONE, "launch_log100_check", [&] { return launch_log100_check(lo, hi, bad, h->stream); });
    return c.finish();
}

// test hook: number of (re, im) pairs of index [lo, hi) for which the MFCC kernels' magnitude step differs from IEEE
// (u32)(sqrtf(pw) * 10); which = 0: mag10_small, i < 16419^2; which = 1: mag10, i < 2^32 (must be 0 over each domain)
int sr_debug_mag10_mismatches(sr_handle *h, int which, uint64_t lo, uint64_t hi, uint64_t *mismatches) {
    SR_REQUIRE(h, h && mismatches && (which == 0 || which == 1) && hi <= (which ? 1ull << 32 : 16419ull * 16419ull));
    HostCall c(h, "sr_debug_mag10_mismatches");
    auto *bad = reinterpret_cast<unsigned long long *>(c.out(h->scratch[2], mismatches, 8, 8));
    c.ck("cudaMemsetAsync", bad ? cudaMemsetAsync(bad, 0, 8, h->stream) : cudaSuccess);
    c.launch(TAG_NONE, "launch_mag10_check", [&] { return launch_mag10_check(which, lo, hi, bad, h->stream); });
    return c.finish();
}

}  // extern "C"

// ---- (1) the reference's own entry points: batch-of-1 on a lazily created default handle -----------
static std::mutex g_default_mu;
static sr_handle *g_default = nullptr;

// f(default handle) under the default handle's lock, created on first use; `none` when there is no device
template <class R, class F> static R on_default_handle(R none, F f) {
    std::lock_guard<std::mutex> lk(g_default_mu);
    if (!g_default) {
        sr_handle *h = nullptr;
        if (sr_create(0, &h) == 0) g_default = h;
    }
    return g_default ? f(g_default) : none;
}

extern "C" {

// VAD.H:24 / VAD.C:22-71. On failure (no device) *atap is left untouched and sr_last_error(NULL) is set.
void noise_atap(const uint16_t *noise, uint16_t n_len, atap_tag *atap) {
    on_default_handle(0, [&](sr_handle *h) { return noise && atap && n_len ? sr_noise_atap_batch(h, noise, n_len, 1, n_len, atap) : 0; });
}

// VAD.H:25 / VAD.C:97-218. Segments come back as pointers into the caller's buffer.
void VAD(const uint16_t *vc, uint16_t buf_len, valid_tag *valid_voice, atap_tag *atap_arg) {
    if (valid_voice) for (unsigned i = 0; i < SR_MAX_VC_CON; ++i) { valid_voice[i].start = nullptr; valid_voice[i].end = nullptr; }   // VAD.C:115-119
    uint32_t seg[6];
    if (on_default_handle(-1, [&](sr_handle *h) {
            return vc && valid_voice && atap_arg && buf_len ? sr_vad_batch(h, vc, buf_len, 1, buf_len, atap_arg, seg) : -1;
        }) != 0) return;
    for (unsigned i = 0; i < SR_MAX_VC_CON; ++i) {
        valid_voice[i].start = seg[2 * i] == SR_SEG_NULL ? nullptr : const_cast<uint16_t *>(vc) + seg[2 * i];
        valid_voice[i].end = seg[2 * i + 1] == SR_SEG_NULL ? nullptr : const_cast<uint16_t *>(vc) + seg[2 * i + 1];
    }
}

// MFCC.H:27 / MFCC.C:86-191. Like the reference this reads valid->start[-1] (MFCC.C:119, i=0).
void get_mfcc(valid_tag *valid, v_ftr_tag *v_ftr, atap_tag *atap_arg) {
    if (!v_ftr) return;
    const int rc = on_default_handle(-1, [&](sr_handle *h) {
        if (!valid || !atap_arg || !valid->start || !valid->end || valid->end < valid->start) return -1;
        // more than vv_frm_max frames is rejected by the kernel (MFCC.C:103-107); cap what is shipped to the device
        const size_t len = std::min((size_t)(valid->end - valid->start), (size_t)(120 * 80 + 80));
        const uint32_t U = (uint32_t)len + 1;
        const uint32_t seg[2] = {1u, U};
        return sr_mfcc_batch(h, valid->start - 1, U, 1, seg, 2, atap_arg, v_ftr);
    });
    if (rc != 0) v_ftr->frm_num = 0;
}

// the reference keeps in_frm_num / mdl_frm_num of the last dtw() call in file statics (DTW.C:65-68, set at :130-131);
// dtw_limit() reads them. Here they are per calling thread.
static thread_local uint16_t g_last_I = 0, g_last_M = 0;

// DTW.C:76-109 (global, no header): 0 = "ins", 1 = "outs", for the (I, M) of this thread's last dtw() call
uint8_t dtw_limit(uint16_t x, uint16_t y) {
    return on_default_handle<uint8_t>(1, [&](sr_handle *h) -> uint8_t {
        uint8_t r = 1;
        return sr_dtw_limit_batch(h, &x, &y, &g_last_I, &g_last_M, 1, &r) == 0 ? r : 1;
    });
}

// DTW.H:7 / DTW.C:120-192: the scan of sr_dtw_batch against a one-slot bank holding frt_mdl
uint32_t dtw(v_ftr_tag *ftr_in, v_ftr_tag *frt_mdl) {
    return on_default_handle<uint32_t>(SR_DIS_ERR, [&](sr_handle *h) -> uint32_t {
        if (!ftr_in || !frt_mdl) return SR_DIS_ERR;
        g_last_I = ftr_in->frm_num; g_last_M = frt_mdl->frm_num;                  // DTW.C:130-131
        uint32_t score = SR_DIS_ERR;
        HostCall c(h, "dtw");
        const BankView one = {c.in(h->scratch[2], frt_mdl, kFtrBytes, 16), 1, (u32)kFtrBytes, nullptr};
        return dtw_host(c, one, ftr_in, 1, 0, 0, &score, nullptr, nullptr) == 0 ? score : SR_DIS_ERR;
    });
}

// MFCC.C:27-62: returns a pointer to a buffer owned by the library (thread-local instead of the
// reference's single static): [0,512) magnitudes, [512,1024) the raw packed FFT bins like fft_out.
uint32_t *fft(int16_t *dat_buf, uint16_t buf_len) {
    static thread_local uint32_t out[SR_FFT_POINT];
    if (buf_len > SR_FFT_POINT || !dat_buf) return nullptr;          // MFCC.C:32-35
    return on_default_handle<uint32_t *>(nullptr, [&](sr_handle *h) -> uint32_t * {
        HostCall c(h, "fft");                                        // all raw bins, then the magnitudes over [0, 512)
        return fft_host(c, nullptr, dat_buf, buf_len, 1, out, out) == 0 ? out : nullptr;
    });
}

// DTW.C:45-62
uint32_t get_dis(int16_t *frm_ftr1, int16_t *frm_ftr2) {
    return on_default_handle<uint32_t>(SR_DIS_ERR, [&](sr_handle *h) -> uint32_t {
        uint32_t d = SR_DIS_ERR;
        return frm_ftr1 && frm_ftr2 && sr_get_dis_batch(h, frm_ftr1, frm_ftr2, 1, &d) == 0 ? d : SR_DIS_ERR;
    });
}

}  // extern "C"
