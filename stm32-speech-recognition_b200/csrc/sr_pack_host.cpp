// sr_pack_host.cpp -- host side of the packed PCM transport of sr_recognise_batch (sr_api.cu).
//
// The end-to-end call is bound by the PCIe copy of the u16 PCM (1.05 GB per 65 536 utterances, ~54 GB/s). The
// reference's samples are 12-bit ADC readings (ADC.C: 12-bit right-aligned conversions), so host worker threads
// repack chunks whose samples are all < 4096 into 12 bits per sample (3 bytes per sample pair: a | b << 12,
// little endian) while other chunks travel unpacked; the device expands them again before the first kernel
// (unpack12_kernel). Any chunk holding a sample >= 4096 is sent as it is, so the call stays exact for every u16
// input. Plain C++ (built with g++, not nvcc) so that the SIMD variants can use target attributes.
#include <immintrin.h>
#include <x86intrin.h>
#include <sched.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>
#include <atomic>
#include <condition_variable>
#include <mutex>
#include <thread>
#include <vector>
#include "sr_pack_host.h"

namespace srk {

// ---- 12-bit packing of n samples (n even); returns the OR of all samples (valid iff (result & 0xF000) == 0) -------
static uint32_t pack12_scalar(const uint16_t *src, size_t n, uint8_t *dst) {
    uint32_t o = 0;
    for (size_t i = 0; i + 2 <= n; i += 2) {
        const uint32_t a = src[i], b = src[i + 1];
        o |= a | b;
        uint8_t *d = dst + (i >> 1) * 3;
        d[0] = (uint8_t)a;
        d[1] = (uint8_t)((a >> 8) | (b << 4));
        d[2] = (uint8_t)(b >> 4);
    }
    return o;
}

__attribute__((target("avx2"))) static uint32_t pack12_avx2(const uint16_t *src, size_t n, uint8_t *dst) {
    const __m256i m1 = _mm256_set1_epi32(0x00000FFF), m2 = _mm256_set1_epi32(0x00FFF000);
    const __m256i shuf = _mm256_setr_epi8(0, 1, 2, 4, 5, 6, 8, 9, 10, 12, 13, 14, -1, -1, -1, -1,
                                          0, 1, 2, 4, 5, 6, 8, 9, 10, 12, 13, 14, -1, -1, -1, -1);
    const __m256i perm = _mm256_setr_epi32(0, 1, 2, 4, 5, 6, 3, 7);
    __m256i acc = _mm256_setzero_si256();
    size_t i = 0;
    for (; i + 16 <= n; i += 16) {
        const __m256i v = _mm256_loadu_si256(reinterpret_cast<const __m256i *>(src + i));
        acc = _mm256_or_si256(acc, v);
        // per 32-bit lane (a | b << 16): 24 bits a | b << 12
        const __m256i p = _mm256_or_si256(_mm256_and_si256(v, m1), _mm256_and_si256(_mm256_srli_epi32(v, 4), m2));
        const __m256i r = _mm256_permutevar8x32_epi32(_mm256_shuffle_epi8(p, shuf), perm);   // 24 bytes at the bottom
        uint8_t *d = dst + (i >> 1) * 3;
        _mm_storeu_si128(reinterpret_cast<__m128i *>(d), _mm256_castsi256_si128(r));
        _mm_storel_epi64(reinterpret_cast<__m128i *>(d + 16), _mm256_extracti128_si256(r, 1));
    }
    uint32_t lanes[8];
    _mm256_storeu_si256(reinterpret_cast<__m256i *>(lanes), acc);
    uint32_t o = 0;
    for (int k = 0; k < 8; ++k) o |= lanes[k];
    o = (o | (o >> 16)) & 0xFFFFu;
    return o | pack12_scalar(src + i, n - i, dst + (i >> 1) * 3);
}

__attribute__((target("avx512f,avx512bw,avx512vbmi"))) static uint32_t pack12_vbmi(const uint16_t *src, size_t n,
                                                                                   uint8_t *dst) {
    alignas(64) static const uint8_t idxb[64] = {0,  1,  2,  4,  5,  6,  8,  9,  10, 12, 13, 14, 16, 17, 18, 20,
                                                 21, 22, 24, 25, 26, 28, 29, 30, 32, 33, 34, 36, 37, 38, 40, 41,
                                                 42, 44, 45, 46, 48, 49, 50, 52, 53, 54, 56, 57, 58, 60, 61, 62,
                                                 0,  0,  0,  0,  0,  0,  0,  0,  0,  0,  0,  0,  0,  0,  0,  0};
    const __m512i idx = _mm512_load_si512(idxb);
    const __m512i m1 = _mm512_set1_epi32(0x00000FFF), m2 = _mm512_set1_epi32(0x00FFF000);
    __m512i acc = _mm512_setzero_si512();
    size_t i = 0;
    for (; i + 32 <= n; i += 32) {
        const __m512i v = _mm512_loadu_si512(src + i);
        acc = _mm512_or_si512(acc, v);
        const __m512i p = _mm512_or_si512(_mm512_and_si512(v, m1), _mm512_and_si512(_mm512_srli_epi32(v, 4), m2));
        _mm512_mask_storeu_epi8(dst + (i >> 1) * 3, 0xFFFFFFFFFFFFull, _mm512_permutexvar_epi8(idx, p));
    }
    uint32_t o = (uint32_t)_mm512_reduce_or_epi32(acc);
    o = (o | (o >> 16)) & 0xFFFFu;
    return o | pack12_scalar(src + i, n - i, dst + (i >> 1) * 3);
}

// Same, 128 samples (three whole cache lines of output) per iteration with two-source byte permutes and NON-TEMPORAL
// stores: the packed bytes go straight to memory without the read-for-ownership a normal store to a cold line costs
// (2 B read + 1.5 B written per sample instead of 2 + 1.5 + 1.5). dst must be 64-byte aligned.
__attribute__((target("avx512f,avx512bw,avx512vbmi"))) static uint32_t pack12_vbmi_nt(const uint16_t *src, size_t n,
                                                                                      uint8_t *dst) {
    if (reinterpret_cast<uintptr_t>(dst) & 63) return pack12_vbmi(src, n, dst);
    alignas(64) uint8_t i0[64], i1[64], i2[64];
    auto at = [](int k) { return (uint8_t)(4 * (k / 3) + k % 3); };          // packed byte k of a vector -> byte of the 24-in-32 layout
    for (int j = 0; j < 64; ++j) {
        i0[j] = j < 48 ? at(j) : (uint8_t)(64 + at(j - 48));                   // line 0: vector 0 bytes 0..47, vector 1 bytes 0..15
        i1[j] = j < 32 ? at(16 + j) : (uint8_t)(64 + at(j - 32));              // line 1: vector 1 bytes 16..47, vector 2 bytes 0..31
        i2[j] = j < 16 ? at(32 + j) : (uint8_t)(64 + at(j - 16));              // line 2: vector 2 bytes 32..47, vector 3 bytes 0..47
    }
    const __m512i x0 = _mm512_load_si512(i0), x1 = _mm512_load_si512(i1), x2 = _mm512_load_si512(i2);
    const __m512i m1 = _mm512_set1_epi32(0x00000FFF), m2 = _mm512_set1_epi32(0x00FFF000);
    __m512i acc = _mm512_setzero_si512();
    size_t i = 0;
    for (; i + 128 <= n; i += 128) {
        const __m512i v0 = _mm512_loadu_si512(src + i), v1 = _mm512_loadu_si512(src + i + 32),
                      v2 = _mm512_loadu_si512(src + i + 64), v3 = _mm512_loadu_si512(src + i + 96);
        acc = _mm512_or_si512(_mm512_or_si512(acc, _mm512_or_si512(v0, v1)), _mm512_or_si512(v2, v3));
        const __m512i p0 = _mm512_or_si512(_mm512_and_si512(v0, m1), _mm512_and_si512(_mm512_srli_epi32(v0, 4), m2));
        const __m512i p1 = _mm512_or_si512(_mm512_and_si512(v1, m1), _mm512_and_si512(_mm512_srli_epi32(v1, 4), m2));
        const __m512i p2 = _mm512_or_si512(_mm512_and_si512(v2, m1), _mm512_and_si512(_mm512_srli_epi32(v2, 4), m2));
        const __m512i p3 = _mm512_or_si512(_mm512_and_si512(v3, m1), _mm512_and_si512(_mm512_srli_epi32(v3, 4), m2));
        uint8_t *d = dst + (i >> 1) * 3;
        _mm512_stream_si512(reinterpret_cast<__m512i *>(d), _mm512_permutex2var_epi8(p0, x0, p1));
        _mm512_stream_si512(reinterpret_cast<__m512i *>(d + 64), _mm512_permutex2var_epi8(p1, x1, p2));
        _mm512_stream_si512(reinterpret_cast<__m512i *>(d + 128), _mm512_permutex2var_epi8(p2, x2, p3));
    }
    _mm_sfence();
    uint32_t o = (uint32_t)_mm512_reduce_or_epi32(acc);
    o = (o | (o >> 16)) & 0xFFFFu;
    return o | pack12_vbmi(src + i, n - i, dst + (i >> 1) * 3);
}

typedef uint32_t (*pack_fn)(const uint16_t *, size_t, uint8_t *);
static pack_fn pick_pack() {
    __builtin_cpu_init();
    if (__builtin_cpu_supports("avx512vbmi") && __builtin_cpu_supports("avx512bw")) return pack12_vbmi_nt;
    if (__builtin_cpu_supports("avx2")) return pack12_avx2;
    return pack12_scalar;
}
uint32_t pack12(const uint16_t *src, size_t n, uint8_t *dst) {
    static const pack_fn f = pick_pack();
    return f(src, n, dst);
}
uint32_t pack12_variant(int variant, const uint16_t *src, size_t n, uint8_t *dst) {
    __builtin_cpu_init();
    const bool vbmi = __builtin_cpu_supports("avx512vbmi") && __builtin_cpu_supports("avx512bw");
    if (variant == 3 && vbmi) return pack12_vbmi_nt(src, n, dst);
    if (variant == 2 && vbmi) return pack12_vbmi(src, n, dst);
    if (variant == 1 && __builtin_cpu_supports("avx2")) return pack12_avx2(src, n, dst);
    if (variant == 0) return pack12_scalar(src, n, dst);
    return 0xFFFFFFFFu;   // variant not available on this CPU
}

// CPUs this process may use: affinity mask capped by the cgroup CPU quota (cpu.max: "quota period" or "max")
int usable_cpus() {
    cpu_set_t set;
    int n = 1;
    if (sched_getaffinity(0, sizeof set, &set) == 0) n = CPU_COUNT(&set);
    FILE *f = fopen("/sys/fs/cgroup/cpu.max", "r");
    if (f) {
        char q[64];
        long long period = 0;
        if (fscanf(f, "%63s %lld", q, &period) == 2 && strcmp(q, "max") != 0 && period > 0) {
            const long long quota = atoll(q);
            const int cap = (int)((quota + period - 1) / period);
            if (cap >= 1 && cap < n) n = cap;
        }
        fclose(f);
    }
    return n < 1 ? 1 : n;
}

// ---- fork-join pool: run() packs one range with all workers ---------------------------------------------------------
// The pool is used in bursts (one fork-join per 32 MB chunk, back to back for the duration of one sr_recognise_batch
// call), so workers SPIN briefly for the next job before they go to sleep on the condition variable: a futex wake-up
// per worker per chunk (~50 us each way) would cost as much as packing the chunk. The caller of run() packs a slice
// itself instead of idling.
struct PackPool::Impl {
    std::vector<std::thread> th;
    std::mutex m;
    std::condition_variable cv_go;
    std::atomic<uint64_t> gen{0};
    std::atomic<int> remaining{0};
    std::atomic<int> sleepers{0};
    std::atomic<bool> stop{false};
    const uint16_t *src = nullptr;
    uint8_t *dst = nullptr;
    size_t n = 0;
    std::atomic<uint32_t> orbits{0};
    int nthreads = 0;                                   // slices per job = workers + the caller

    void slice(int t) {
        // slices are multiples of 128 samples (192 packed bytes, three cache lines): no two workers touch the same line
        const size_t groups = n / 128, per = (groups + nthreads - 1) / nthreads;
        const size_t g0 = (size_t)t * per, g1 = g0 + per < groups ? g0 + per : groups;
        uint32_t o = 0;
        if (g0 < g1) o = pack12(src + g0 * 128, (g1 - g0) * 128, dst + g0 * 192);
        if (t == nthreads - 1 && groups * 128 < n) o |= pack12(src + groups * 128, n - groups * 128, dst + groups * 192);
        orbits.fetch_or(o, std::memory_order_relaxed);
    }
    void worker(int t) {
        uint64_t seen = 0;
        for (;;) {
            bool got = false;
            const uint64_t t0 = __rdtsc();
            while (!got) {                                               // poll ~150 us (at ~2-3 GHz TSC) between chunks
                if (stop.load(std::memory_order_acquire)) return;
                if (gen.load(std::memory_order_acquire) != seen) got = true;
                else if (__rdtsc() - t0 > 400000ull) break;
                else _mm_pause();
            }
            if (!got) {
                std::unique_lock<std::mutex> lk(m);
                sleepers.fetch_add(1, std::memory_order_relaxed);
                cv_go.wait(lk, [&] { return stop.load(std::memory_order_acquire) || gen.load(std::memory_order_acquire) != seen; });
                sleepers.fetch_sub(1, std::memory_order_relaxed);
                if (stop.load(std::memory_order_acquire)) return;
            }
            seen = gen.load(std::memory_order_acquire);
            slice(t);
            remaining.fetch_sub(1, std::memory_order_acq_rel);
        }
    }
};

PackPool::PackPool(int nthreads) : p(new Impl) {
    p->nthreads = nthreads < 1 ? 1 : nthreads;
    for (int t = 1; t < p->nthreads; ++t) p->th.emplace_back([this, t] { p->worker(t); });   // slice 0 is the caller's
}
PackPool::~PackPool() {
    {
        std::lock_guard<std::mutex> lk(p->m);
        p->stop.store(true, std::memory_order_release);
    }
    p->cv_go.notify_all();
    for (auto &t : p->th) t.join();
    delete p;
}
int PackPool::threads() const { return p->nthreads; }
uint32_t PackPool::run(const uint16_t *src, size_t n, uint8_t *dst) {
    p->src = src; p->dst = dst; p->n = n;
    p->orbits.store(0, std::memory_order_relaxed);
    p->remaining.store(p->nthreads - 1, std::memory_order_relaxed);
    {
        std::lock_guard<std::mutex> lk(p->m);                          // pairs with the sleepers' predicate check
        p->gen.fetch_add(1, std::memory_order_release);
    }
    if (p->sleepers.load(std::memory_order_relaxed) > 0) p->cv_go.notify_all();
    p->slice(0);
    while (p->remaining.load(std::memory_order_acquire) != 0) _mm_pause();
    return p->orbits.load(std::memory_order_relaxed);
}

}  // namespace srk
