// sr_transport.cu -- the packed PCM transport of sr_recognise_batch (sr_api.cu): whether a call packs, the worker pool
// and the staging that pack, the send loop that interleaves packed and plain chunks, and the automatic mode's
// measurements. What one chunk does on the device (copy, expansion, kernels) is the caller's step.
#include "sr_internal.h"
#include <condition_variable>
#include <deque>
#include <utility>
#include "sr_pack_host.h"
#include "sr_numa.h"

// ranks of this node that share the host (torchrun exports LOCAL_WORLD_SIZE)
static int local_world_size() {
    static const int local_world = [] { const char *e = getenv("LOCAL_WORLD_SIZE"); const int v = e ? atoi(e) : 1; return v > 0 ? v : 1; }();
    return local_world;
}
// CPUs this rank may count on: the process' usable CPUs (affinity capped by the cgroup quota) divided by those ranks
static int rank_cpu_share() { return usable_cpus() / local_world_size(); }

// local ranks whose GPU hangs off the same NUMA node as this handle's (torchrun convention: local rank r drives device r);
// unknown topology counts everybody
static int ranks_on_socket(const sr_handle *h) {
    const int W = local_world_size();
    if (W <= 1) return 1;
    if (h->numa_node < 0) return W;
    int n = 0;
    for (int d = 0; d < W; ++d) if (sr_device_numa_node(d) == h->numa_node) ++n;
    return n < 1 ? 1 : n;
}

// samples of chunk c: `chunk` utterances of U samples, fewer in the last chunk
static size_t chunk_samples(uint32_t c, uint32_t chunk, uint32_t U, uint32_t B) {
    const uint32_t b0 = c * chunk;
    return (size_t)(b0 + chunk <= B ? chunk : B - b0) * U;
}

// 1 = forced on, 0 = forced off, -1 = automatic (decided per call by auto_pick)
int PackedTransport::resolved_mode(const sr_handle *h) const {
    int m = mode;
    if (m < 0) {
        static const int env_mode = [] { const char *e = getenv("SR_PACK12"); return e && *e ? atoi(e) : -1; }();
        m = env_mode;
    }
    // automatic: needs CPUs to pack with, and the socket's DRAM bandwidth to itself: with several GPUs per socket the DMA
    // reads alone load it (4 x 54 GB/s at four) and packing measured 25.8 vs 19.5 ms at 4 and 8 ranks, 19.8-21.3 vs 19.5 with
    // two ranks on one socket -- and ranks that probe at different moments talk each other into it. One rank per socket only.
    if (m < 0 && !(rank_cpu_share() >= 6 && ranks_on_socket(h) <= 1)) m = 0;
    return m;
}

// Automatic mode measures instead of guessing. Whether packing pays depends on what else loads the host's memory system:
// one or two ranks per socket gain ~16 % (16.3 vs 19.4 ms per 1.05 GB), but with four ranks per socket the DMA reads
// alone take ~216 GB/s of that socket's DRAM bandwidth and the packers' extra traffic makes the call SLOWER (25.8 vs
// 19.5 ms, measured at 4 and 8 GPUs). So: the first qualifying call goes plain, the second packed, then the faster of
// the two (ns per byte, exponentially averaged; packing must win by 7 %) is used, with the other re-probed every 32nd call.
// With more than one rank on this GPU's socket the automatic mode stays plain (resolved_mode above).
bool PackedTransport::auto_pick() {
    const uint64_t n = auto_calls++;
    if (auto_ns_per_byte[0] <= 0.0) return false;
    if (auto_ns_per_byte[1] <= 0.0) return true;
    const bool packed_better = auto_ns_per_byte[1] < 0.93 * auto_ns_per_byte[0];   // a clear win only (N = 1: 0.84)
    if (n % 32 == 31) return !packed_better;                       // probe the loser now and then: conditions change
    return packed_better;
}

void PackedTransport::call_done(uint64_t pcm_bytes) {
    if (!probe) return;
    const double ns_per_byte = std::chrono::duration<double, std::nano>(std::chrono::steady_clock::now() - t_call0).count() / (double)pcm_bytes;
    double &v = auto_ns_per_byte[last_packed > 0 ? 1 : 0];   // a packed call whose chunks all went plain counts as plain
    v = v <= 0.0 ? ns_per_byte : 0.75 * v + 0.25 * ns_per_byte;
}

PackedTransport::~PackedTransport() = default;

// workers, pinned staging slots of pk bytes, device staging; false (CUDA error cleared) = send this call plain
bool PackedTransport::setup(const sr_handle *h, size_t pk) {
    ScopedNodeAffinity node_scope(h->numa_node);          // workers inherit it; staging pages are allocated from this node
    if (!pool) {
        // packers = this rank's CPU share minus room for the sender, the CUDA runtime's threads and the caller's own work
        static const int env_nt = [] { const char *e = getenv("SR_PACK_THREADS"); return e && *e ? atoi(e) : 0; }();
        // (measured on a 2 x 32-core host, 16-CPU quota: 8..12 packers all land at ~16.3 ms per 1.05 GB step; more only add
        // memory traffic next to the DMA reads, which slows the link: 54 -> 47 GB/s at 14 packers)
        int nt = env_nt > 0 ? env_nt : rank_cpu_share() - 3;
        if (env_nt <= 0 && nt > 10) nt = 10;
        nt = nt > 16 ? 16 : nt;
        if (nt >= 2) pool.reset(new (std::nothrow) PackPool(nt));
    }
    if (pool && stage_cap < pk) {
        for (auto &st : stage) st.reset();
        stage_cap = 0;
        bool ok = true;
        for (auto &st : stage) if (ok && st.alloc(pk) != cudaSuccess) ok = false;
        if (ok) stage_cap = pk;
        else { cudaGetLastError(); for (auto &st : stage) st.reset(); }
    }
    if (!pool || !stage_cap || ensure(dpacked, 2 * stage_cap) != cudaSuccess) { cudaGetLastError(); return false; }
    return true;
}

int PackedTransport::send(sr_handle *h, const uint16_t *pcm, uint32_t U, uint32_t B, uint32_t chunk, const Step &step) {
    const uint32_t nchunks = (B + chunk - 1) / chunk;
    last_packed = 0; last_plain = 0; last_h2d = 0;
    const int tmode = nchunks >= 4 ? resolved_mode(h) : 0;
    const bool tauto = tmode < 0;
    bool packed = tmode > 0 || (tauto && auto_pick());
    t_call0 = std::chrono::steady_clock::now();
    bool did_setup = false;                               // this call created the pool / staging: its time is not a measurement
    if (packed) {
        const size_t pk = ((((size_t)chunk * U + 1) / 2 * 3 + 64 + 255) / 256) * 256;
        did_setup = !pool || stage_cap < pk || dpacked.cap < 2 * pk;
        packed = setup(h, pk);
    }
    probe = tauto && !did_setup;
    if (packed) return send_packed(h, pcm, U, B, chunk, step);
    for (uint32_t c = 0; c < nchunks; ++c) {
        const int rc = step(c, (int)(c & 1), nullptr);
        if (rc) return rc;
        last_h2d += chunk_samples(c, chunk, U, B) * 2; ++last_plain;
    }
    return 0;
}

// The caller's thread sends chunks from the front as plain u16, paced by the copy engine; the worker pool packs chunks
// from the back into the staging slots and those are sent packed as soon as they are ready. The two meet in the middle,
// so the call is never slower than the plain path and approaches 3/4 of its PCIe time.
int PackedTransport::send_packed(sr_handle *h, const uint16_t *pcm, uint32_t U, uint32_t B, uint32_t chunk, const Step &step) {
    const uint32_t nchunks = (B + chunk - 1) / chunk;
    std::mutex m;
    std::condition_variable cv_slot;
    std::deque<std::pair<uint32_t, int>> ready;           // (chunk, staging slot)
    std::vector<uint32_t> retry;                          // chunks that hold a sample >= 4096: sent plain
    int lo = 0, hi = (int)nchunks - 1;                    // unclaimed chunks [lo, hi]
    unsigned free_mask = (1u << kStage) - 1u;
    bool abort = false;
    std::thread packer([&] {
        ScopedNodeAffinity bind(h->numa_node);            // slice 0 of every chunk is packed by this thread
        for (;;) {
            int slot;
            uint32_t c;
            {
                std::unique_lock<std::mutex> lk(m);
                cv_slot.wait(lk, [&] { return abort || lo > hi || free_mask != 0; });
                if (abort || lo > hi) return;
                slot = __builtin_ctz(free_mask);
                free_mask &= ~(1u << slot);
                c = (uint32_t)hi--;
            }
            const size_t ns = chunk_samples(c, chunk, U, B);
            const uint32_t orb = (ns & 1) ? 0xFFFFu : pool->run(pcm + (size_t)c * chunk * U, ns, stage[slot].p);
            {
                std::lock_guard<std::mutex> lk(m);
                if (orb & 0xF000u) { retry.push_back(c); free_mask |= 1u << slot; }
                else ready.emplace_back(c, slot);
            }
        }
    });
    int rc = 0;
    int slot_of[2] = {-1, -1};                            // staging slot behind the copy last issued on each buffer
    auto release = [&](int &sl) {
        if (sl < 0) return;
        { std::lock_guard<std::mutex> lk(m); free_mask |= 1u << sl; }
        cv_slot.notify_one();
        sl = -1;
    };
    uint32_t sent = 0;
    while (sent < nchunks) {
        int slot = -1;
        long c = -1;
        {
            std::lock_guard<std::mutex> lk(m);
            if (!ready.empty()) { c = ready.front().first; slot = ready.front().second; ready.pop_front(); }
            else if (!retry.empty()) { c = retry.back(); retry.pop_back(); }
            else if (lo <= hi) c = lo++;
        }
        if (c < 0) { std::this_thread::sleep_for(std::chrono::microseconds(50)); continue; }   // every chunk is claimed; the pool is still packing
        const int buf = (int)(sent & 1);
        if (sent >= 2) {                                               // at most two copies in flight: paces this thread
            cudaError_t e = cudaEventSynchronize(h->ev_h2d[buf]);
            if (e != cudaSuccess) { rc = fail(h, "cudaEventSynchronize", e); if (slot >= 0) release(slot); break; }
            release(slot_of[buf]);
        }
        rc = step((uint32_t)c, buf, slot >= 0 ? stage[slot].p : nullptr);
        if (rc) { if (slot >= 0) release(slot); break; }
        const size_t ns = chunk_samples((uint32_t)c, chunk, U, B);
        if (slot >= 0) { last_h2d += ns / 2 * 3; ++last_packed; }
        else { last_h2d += ns * 2; ++last_plain; }
        slot_of[buf] = slot;
        ++sent;
    }
    { std::lock_guard<std::mutex> lk(m); abort = true; }
    cv_slot.notify_all();
    packer.join();
    if (rc) { cudaStreamSynchronize(h->copy_stream); return rc; }
    return 0;
}
