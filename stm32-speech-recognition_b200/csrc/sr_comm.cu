// sr_comm.cu -- the one exchange step of the path behind the C-ABI (SURVEY 8e, 8b(3)): utterances are sharded over
// ranks (one handle per GPU, one process or one thread per rank) and the per-template scores -- plus the 8-byte
// (distance, index) argmin keys -- of all shards are all-gathered over NCCL, so that a C host needs no Python and no
// torch for the multi-GPU form of spch_recg (main.c:249-296).
//
// NCCL is bound at run time (dlopen of libnccl.so.2: the copy already loaded into the process -- e.g. torch's -- or the
// system one), so libspeech_b200.so itself has no link-time dependency on it and single-GPU users never load it.
// The collective runs on a stream of its own: it starts when the kernels that produced the scores have finished and
// overlaps whatever the handle's stream does next (the next batch's VAD/MFCC); the next writer of the same score
// buffer and sr_comm_wait / sr_sync order themselves after it with events.
#include "sr_internal.h"
#include <dlfcn.h>

namespace {

// the slice of nccl.h this file needs (types are ABI-stable across NCCL 2.x)
typedef struct { char internal[128]; } ncclUniqueId_t;
typedef void *ncclComm_p;
enum { kNcclUint8 = 1 };
struct NcclApi {
    void *lib = nullptr;
    int (*GetUniqueId)(ncclUniqueId_t *) = nullptr;
    int (*CommInitRank)(ncclComm_p *, int, ncclUniqueId_t, int) = nullptr;
    int (*CommDestroy)(ncclComm_p) = nullptr;
    int (*AllGather)(const void *, void *, size_t, int, ncclComm_p, cudaStream_t) = nullptr;
    const char *(*GetErrorString)(int) = nullptr;
    int (*GetVersion)(int *) = nullptr;
    int (*GroupStart)() = nullptr;
    int (*GroupEnd)() = nullptr;
    std::string why;
};

NcclApi *nccl_api() {
    static NcclApi api;
    static std::once_flag once;
    std::call_once(once, [] {
        const char *env = getenv("SR_NCCL_LIB");
        const char *names[] = {env, "libnccl.so.2", "libnccl.so"};
        for (const char *n : names) {
            if (!n || !*n) continue;
            api.lib = dlopen(n, RTLD_NOW | RTLD_GLOBAL);
            if (api.lib) break;
        }
        if (!api.lib) { api.why = "libnccl.so.2 not found (set SR_NCCL_LIB)"; return; }
        auto sym = [&](const char *s) { void *p = dlsym(api.lib, s); if (!p) api.why = std::string("missing NCCL symbol ") + s; return p; };
        api.GetUniqueId = reinterpret_cast<int (*)(ncclUniqueId_t *)>(sym("ncclGetUniqueId"));
        api.CommInitRank = reinterpret_cast<int (*)(ncclComm_p *, int, ncclUniqueId_t, int)>(sym("ncclCommInitRank"));
        api.CommDestroy = reinterpret_cast<int (*)(ncclComm_p)>(sym("ncclCommDestroy"));
        api.AllGather = reinterpret_cast<int (*)(const void *, void *, size_t, int, ncclComm_p, cudaStream_t)>(sym("ncclAllGather"));
        api.GetErrorString = reinterpret_cast<const char *(*)(int)>(sym("ncclGetErrorString"));
        api.GetVersion = reinterpret_cast<int (*)(int *)>(sym("ncclGetVersion"));
        api.GroupStart = reinterpret_cast<int (*)()>(sym("ncclGroupStart"));
        api.GroupEnd = reinterpret_cast<int (*)()>(sym("ncclGroupEnd"));
    });
    return &api;
}

int nccl_fail(sr_handle *h, const char *what, int rc) {
    NcclApi *a = nccl_api();
    char buf[384];
    snprintf(buf, sizeof buf, "%s: NCCL error %d (%s)", what, rc, (a->GetErrorString && rc > 0) ? a->GetErrorString(rc) : a->why.c_str());
    g_tls_error = buf;
    if (h) h->err = buf;
    return rc > 0 ? 10000 + rc : -2;                               // 10000 + ncclResult_t, or -2: NCCL unavailable
}

}  // namespace

struct sr_comm {
    ncclComm_p comm = nullptr;
    int rank = 0, world = 1;
    cudaStream_t stream = nullptr;                                  // the collective's own stream
    cudaEvent_t ev_ready = nullptr;                                 // producer finished
    // The last two collectives. A recognise call alternates the handle's internal key buffer (best / best_alt) and a caller
    // that alternates its score buffers too never makes the template scan wait for the PREVIOUS batch's gather: the scan
    // only waits for the gather that last read the buffers it is about to rewrite -- two calls back, long finished.
    struct Slot { cudaEvent_t ev_done = nullptr; const void *score = nullptr; bool pending = false; } slot[2];
    int next = 0;                                                   // slot (= key buffer) of the call being issued
};

extern "C" {

int sr_comm_unique_id(void *id128) {
    if (!id128) return fail(nullptr, "sr_comm_unique_id: NULL", cudaSuccess);
    NcclApi *a = nccl_api();
    if (!a->GetUniqueId) return nccl_fail(nullptr, "sr_comm_unique_id", 0);
    ncclUniqueId_t id;
    const int rc = a->GetUniqueId(&id);
    if (rc) return nccl_fail(nullptr, "ncclGetUniqueId", rc);
    memcpy(id128, &id, sizeof id);
    return 0;
}

int sr_comm_nccl_version(void) {
    NcclApi *a = nccl_api();
    int v = 0;
    if (!a->GetVersion || a->GetVersion(&v)) return 0;
    return v;
}

int sr_comm_destroy(sr_handle *h) {
    if (!h || !h->comm) return 0;
    DeviceGuard g(h->device);
    sr_comm *c = h->comm;
    if (c->stream) cudaStreamSynchronize(c->stream);
    if (c->comm) nccl_api()->CommDestroy(c->comm);
    if (c->ev_ready) cudaEventDestroy(c->ev_ready);
    for (auto &sl : c->slot) if (sl.ev_done) cudaEventDestroy(sl.ev_done);
    if (c->stream) cudaStreamDestroy(c->stream);
    delete c;
    h->comm = nullptr;
    return 0;
}

// collective: every rank calls it with the same id (sr_comm_unique_id on one rank, distributed by the host's own means)
int sr_comm_create(sr_handle *h, int rank, int world, const void *id128) {
    SR_REQUIRE(h, h && id128 && world >= 1 && rank >= 0 && rank < world);
    NcclApi *a = nccl_api();
    if (!a->CommInitRank || !a->AllGather || !a->CommDestroy) return nccl_fail(h, "sr_comm_create", 0);
    sr_comm_destroy(h);
    DeviceGuard g(h->device);
    sr_comm *c = new (std::nothrow) sr_comm;
    SR_REQUIRE(h, c != nullptr);
    c->rank = rank; c->world = world;
    h->comm = c;
    // highest priority: when a persistent kernel's CTAs drain, the collective's few CTAs are placed before the next kernel's
    int prio_lo = 0, prio_hi = 0;
    cudaDeviceGetStreamPriorityRange(&prio_lo, &prio_hi);
    cudaError_t e = cudaStreamCreateWithPriority(&c->stream, cudaStreamNonBlocking, prio_hi);
    if (e == cudaSuccess) e = cudaEventCreateWithFlags(&c->ev_ready, cudaEventDisableTiming);
    for (auto &sl : c->slot) if (e == cudaSuccess) e = cudaEventCreateWithFlags(&sl.ev_done, cudaEventDisableTiming);
    if (e != cudaSuccess) { sr_comm_destroy(h); return fail(h, "sr_comm_create: stream/event", e); }
    ncclUniqueId_t id;
    memcpy(&id, id128, sizeof id);
    const int rc = a->CommInitRank(&c->comm, world, id, rank);
    if (rc) { c->comm = nullptr; sr_comm_destroy(h); return nccl_fail(h, "ncclCommInitRank", rc); }
    return 0;
}

int sr_comm_rank(const sr_handle *h) { return h && h->comm ? h->comm->rank : 0; }
int sr_comm_world(const sr_handle *h) { return h && h->comm ? h->comm->world : 1; }

// up to two all-gathers of equal blocks as ONE NCCL group (one kernel): recv[r*bytes .. ) = rank r's send block. Ordered
// after everything issued so far on the handle's stream; runs on the communicator's stream.
static int allgather2(sr_handle *h, const void *send0, void *recv0, size_t bytes0, const void *send1, void *recv1, size_t bytes1,
                      const void *score_tag) {
    sr_comm *c = h->comm;
    NcclApi *a = nccl_api();
    SR_CK(h, cudaEventRecord(c->ev_ready, h->stream));
    SR_CK(h, cudaStreamWaitEvent(c->stream, c->ev_ready, 0));
    const bool group = bytes0 && bytes1 && a->GroupStart && a->GroupEnd;
    int rc = 0;
    if (group) rc = a->GroupStart();
    if (!rc && bytes0) rc = a->AllGather(send0, recv0, bytes0, kNcclUint8, c->comm, c->stream);
    if (!rc && bytes1) rc = a->AllGather(send1, recv1, bytes1, kNcclUint8, c->comm, c->stream);
    if (group) { const int rc2 = a->GroupEnd(); if (!rc) rc = rc2; }
    if (rc) return nccl_fail(h, "ncclAllGather", rc);
    sr_comm::Slot &sl = c->slot[c->next];
    SR_CK(h, cudaEventRecord(sl.ev_done, c->stream));
    sl.pending = true; sl.score = score_tag;
    c->next ^= 1;
    return 0;
}

// All-gather of equal blocks, device pointers (overlaps what the handle's stream does next; see sr_comm_wait)
int sr_allgather_dev(sr_handle *h, const void *send, void *recv, size_t bytes_per_rank) {
    SR_REQUIRE(h, h && h->comm && (bytes_per_rank == 0 || (send && recv)));
    if (bytes_per_rank == 0) return 0;
    DeviceGuard g(h->device);
    return allgather2(h, send, recv, bytes_per_rank, nullptr, nullptr, 0, send);
}

// make the handle's stream wait for the collectives issued so far (then sr_sync / stream order covers them)
int sr_comm_wait(sr_handle *h) {
    SR_REQUIRE(h, h != nullptr);
    if (!h->comm) return 0;
    DeviceGuard g(h->device);
    for (auto &sl : h->comm->slot)
        if (sl.pending) { SR_CK(h, cudaStreamWaitEvent(h->stream, sl.ev_done, 0)); sl.pending = false; }
    return 0;
}

}  // extern "C"

// Before the template scan of a recognise call rewrites score / best: wait for the gathers that may still read them -- the
// one in the slot this call will reuse (it read the same key buffer, two calls ago) and any that read the same score buffer.
int comm_wait_before_scan(sr_handle *h, const void *score) {
    sr_comm *c = h->comm;
    if (!c) return 0;
    h->best_sel = c->next;
    for (int i = 0; i < 2; ++i) {
        sr_comm::Slot &sl = c->slot[i];
        if (sl.pending && (i == c->next || (score && sl.score == score))) {
            SR_CK(h, cudaStreamWaitEvent(h->stream, sl.ev_done, 0));
            sl.pending = false;
        }
    }
    return 0;
}

extern "C" {

// spch_recg for this rank's shard + the exchange step: gathered_score[world*B][n_slot] (u32, rank-major = global
// utterance order for equal shards) and/or gathered_best[world*B] = (best_dis << 32 | best_idx), the key of the
// strict-'<' first-wins argmin (main.c:285-289), or under SR_DTW_KNN(k) of the KNN decision (best_final_kernel<true>
// writes it to the key buffer's first B words). All pointers are device memory; out_dev->score must be non-NULL when
// gathered_score is wanted. Asynchronous: sr_comm_wait + sr_sync (or stream order after sr_comm_wait) to consume.
int sr_recognise_batch_dev_allgather(sr_handle *h, const uint16_t *pcm, uint32_t U, uint32_t B, uint32_t n_len,
                                     const sr_recog_out *out_dev, uint32_t *gathered_score, uint64_t *gathered_best) {
    SR_REQUIRE(h, h && h->comm && out_dev);
    SR_REQUIRE(h, !gathered_score || out_dev->score);
    DeviceGuard g(h->device);
    sr_recog_out o = *out_dev;
    if (gathered_best) SR_CK(h, caller_or_ws(h->bidx, (size_t)B * 4, o.best_idx));   // the argmin forced: keys in key_buf
    // A gather issued earlier may still be reading score / best. Only the template scan rewrites them, so only it waits
    // (comm_wait_before_scan inside recognise_dev_impl) -- and with alternating buffers it waits for the gather of two calls
    // ago, so nothing on the handle's stream ever waits for the previous batch's collective.
    int rc = recognise_dev_impl(h, pcm, U, B, n_len, &o, true);
    if (rc) return rc;
    if (!gathered_score && !gathered_best) return 0;
    const void *keys = key_buf(h).p;                                 // the buffer this call's template scan just filled
    return allgather2(h, gathered_score ? o.score : nullptr, gathered_score, gathered_score ? (size_t)B * h->bank.n * 4 : 0,
                      gathered_best ? keys : nullptr, gathered_best, gathered_best ? (size_t)B * 8 : 0, o.score);
}

}  // extern "C"
