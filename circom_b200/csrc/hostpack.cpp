// Host side of the packed device->host transfer (see hostpack.h).
#include "hostpack.h"

#include <immintrin.h>

#include <pthread.h>
#include <sched.h>

#include <algorithm>
#include <condition_variable>
#include <cstdio>
#include <cstdlib>
#include <mutex>
#include <string>
#include <thread>

namespace cw {

void build_pack_layout(const Tape &t, PackLayout &L, const uint8_t *cls) {
    const size_t W = t.n_witness;
    if (!cls) cls = t.wit_class.data();
    L = PackLayout();
    L.n_plane_words = t.n_bitwords;
    for (size_t i = 0; i < W; ++i) {
        const uint32_t loc = t.witness_slot[i];
        PackSeg sg;
        sg.start = (uint32_t)i;
        sg.count = 1;
        if (loc & OPERAND_BIT) {
            sg.kind = 0;
            sg.src = loc & OPERAND_BITPOS_MASK;
        } else if (cls[i] == 0) {
            sg.kind = 1;
            sg.src = (uint32_t)L.bit_loc.size();
            L.bit_loc.push_back(loc);
        } else if (cls[i] == 1) {
            sg.kind = 2;
            sg.src = (uint32_t)L.u64_loc.size();
            L.u64_loc.push_back(loc);
        } else {
            sg.kind = 3;
            sg.src = (uint32_t)L.full_loc.size();
            L.full_loc.push_back(loc);
        }
        if (!L.segs.empty()) {
            PackSeg &p = L.segs.back();
            // (a plane run stays inside its word)
            const bool same_word = sg.kind != 0 || ((p.src + p.count) >> 5) == (p.src >> 5);
            if (p.kind == sg.kind && p.src + p.count == sg.src && same_word) {
                ++p.count;
                continue;
            }
        }
        L.segs.push_back(sg);
    }
    L.n_bit_words = (L.bit_loc.size() + 31) / 32;
    L.words = (L.n_plane_words + L.n_bit_words + 2 * L.u64_loc.size() + 8 * L.full_loc.size() + 3) & ~(size_t)3;
}

namespace {

// ---- portable (SSE2) ------------------------------------------------------------------------------------------
void expand_sse2(const PackLayout &L, const uint32_t *rec, uint64_t *row_out) {
    const uint32_t *plane = rec, *xb = rec + L.n_plane_words, *pu = xb + L.n_bit_words, *pf = pu + 2 * L.u64_loc.size();
    const bool aligned = (((uintptr_t)row_out) & 15u) == 0;
    const __m128i zero = _mm_setzero_si128();
    auto put = [&](uint64_t *dst, __m128i lo, __m128i hi) {
        if (aligned) {
            _mm_stream_si128((__m128i *)dst, lo);
            _mm_stream_si128((__m128i *)(dst + 2), hi);
        } else {
            _mm_storeu_si128((__m128i *)dst, lo);
            _mm_storeu_si128((__m128i *)(dst + 2), hi);
        }
    };
    for (const PackSeg &sg : L.segs) {
        uint64_t *dst = row_out + 4 * (size_t)sg.start;
        switch (sg.kind) {
            case 0: {
                uint32_t bits = plane[sg.src >> 5] >> (sg.src & 31u);
                for (uint32_t j = 0; j < sg.count; ++j, dst += 4, bits >>= 1)
                    put(dst, _mm_cvtsi64_si128((long long)(bits & 1u)), zero);
                break;
            }
            case 1:
                for (uint32_t j = 0; j < sg.count; ++j, dst += 4) {
                    const uint32_t k = sg.src + j;
                    put(dst, _mm_cvtsi64_si128((long long)((xb[k >> 5] >> (k & 31u)) & 1u)), zero);
                }
                break;
            case 2:
                for (uint32_t j = 0; j < sg.count; ++j, dst += 4)
                    put(dst, _mm_loadl_epi64((const __m128i *)(pu + 2 * (size_t)(sg.src + j))), zero);
                break;
            default:
                for (uint32_t j = 0; j < sg.count; ++j, dst += 4) {
                    const uint32_t *f = pf + 8 * (size_t)(sg.src + j);
                    put(dst, _mm_loadu_si128((const __m128i *)f), _mm_loadu_si128((const __m128i *)(f + 4)));
                }
        }
    }
    _mm_sfence();
}

// (a lambda inside a target("avx2") function is compiled for the base target: a macro instead)
#define put(dst, v)                                                    \
    do {                                                               \
        if (aligned) _mm256_stream_si256((__m256i *)(dst), (v));       \
        else _mm256_storeu_si256((__m256i *)(dst), (v));               \
    } while (0)

// ---- AVX2: one 32-byte streaming store per row ---------------------------------------------------------------------
__attribute__((target("avx2"))) void expand_avx2(const PackLayout &L, const uint32_t *rec, uint64_t *row_out) {
    const uint32_t *plane = rec, *xb = rec + L.n_plane_words, *pu = xb + L.n_bit_words, *pf = pu + 2 * L.u64_loc.size();
    const bool aligned = (((uintptr_t)row_out) & 31u) == 0;
    for (const PackSeg &sg : L.segs) {
        uint64_t *dst = row_out + 4 * (size_t)sg.start;
        switch (sg.kind) {
            case 0: {
                uint32_t bits = plane[sg.src >> 5] >> (sg.src & 31u);
                for (uint32_t j = 0; j < sg.count; ++j, dst += 4, bits >>= 1)
                    put(dst, _mm256_zextsi128_si256(_mm_cvtsi32_si128((int)(bits & 1u))));
                break;
            }
            case 1:
                for (uint32_t j = 0; j < sg.count; ++j, dst += 4) {
                    const uint32_t k = sg.src + j;
                    put(dst, _mm256_zextsi128_si256(_mm_cvtsi32_si128((int)((xb[k >> 5] >> (k & 31u)) & 1u))));
                }
                break;
            case 2:
                for (uint32_t j = 0; j < sg.count; ++j, dst += 4)
                    put(dst, _mm256_zextsi128_si256(_mm_loadl_epi64((const __m128i *)(pu + 2 * (size_t)(sg.src + j)))));
                break;
            default:
                for (uint32_t j = 0; j < sg.count; ++j, dst += 4)
                    put(dst, _mm256_loadu_si256((const __m256i *)(pf + 8 * (size_t)(sg.src + j))));
        }
    }
    _mm_sfence();
}

// ---- AVX-512: plane runs two rows (one cache line) per store ------------------------------------------------------------
__attribute__((target("avx512f,avx512bw,avx512vl,avx2"))) void expand_avx512(const PackLayout &L, const uint32_t *rec,
                                                                              uint64_t *row_out) {
    const uint32_t *plane = rec, *xb = rec + L.n_plane_words, *pu = xb + L.n_bit_words, *pf = pu + 2 * L.u64_loc.size();
    const bool aligned = (((uintptr_t)row_out) & 31u) == 0;
    const __m512i one = _mm512_set1_epi64(1);
    for (const PackSeg &sg : L.segs) {
        uint64_t *dst = row_out + 4 * (size_t)sg.start;
        switch (sg.kind) {
            case 0: {
                uint32_t bits = plane[sg.src >> 5] >> (sg.src & 31u);
                uint32_t j = 0;
                if (aligned && (((uintptr_t)dst) & 63u) && sg.count) {  // reach a cache-line boundary
                    put(dst, _mm256_zextsi128_si256(_mm_cvtsi32_si128((int)(bits & 1u))));
                    dst += 4; bits >>= 1; ++j;
                }
                if (aligned) {
                    // rows 2j, 2j+1 = 64 bytes: qword 0 <- bit 0, qword 4 <- bit 1, everything else zero
                    for (; j + 2 <= sg.count; j += 2, dst += 8, bits >>= 2) {
                        const __mmask8 m = (__mmask8)((bits & 1u) | ((bits & 2u) << 3));
                        _mm512_stream_si512((__m512i *)dst, _mm512_maskz_mov_epi64(m, one));
                    }
                }
                for (; j < sg.count; ++j, dst += 4, bits >>= 1)
                    put(dst, _mm256_zextsi128_si256(_mm_cvtsi32_si128((int)(bits & 1u))));
                break;
            }
            case 1:
                for (uint32_t j = 0; j < sg.count; ++j, dst += 4) {
                    const uint32_t k = sg.src + j;
                    put(dst, _mm256_zextsi128_si256(_mm_cvtsi32_si128((int)((xb[k >> 5] >> (k & 31u)) & 1u))));
                }
                break;
            case 2:
                for (uint32_t j = 0; j < sg.count; ++j, dst += 4)
                    put(dst, _mm256_zextsi128_si256(_mm_loadl_epi64((const __m128i *)(pu + 2 * (size_t)(sg.src + j)))));
                break;
            default:
                for (uint32_t j = 0; j < sg.count; ++j, dst += 4)
                    put(dst, _mm256_loadu_si256((const __m256i *)(pf + 8 * (size_t)(sg.src + j))));
        }
    }
    _mm_sfence();
}

#undef put

int pick_isa() {
    const char *e = getenv("CW_EXPAND_ISA");
    int want = e ? atoi(e) : 512;
    __builtin_cpu_init();
    if (want >= 512 && __builtin_cpu_supports("avx512f") && __builtin_cpu_supports("avx512bw") && __builtin_cpu_supports("avx512vl")) return 2;
    if (want >= 256 && __builtin_cpu_supports("avx2")) return 1;
    return 0;
}
int g_isa = -1;

int env_int(const char *name, int dflt) {
    const char *s = getenv(name);
    return s && *s ? atoi(s) : dflt;
}

}  // namespace

const char *expand_isa() {
    if (g_isa < 0) g_isa = pick_isa();
    return g_isa == 2 ? "avx512" : g_isa == 1 ? "avx2" : "sse2";
}

void expand_record(const PackLayout &L, const uint32_t *rec, uint64_t *row_out, int force_bits) {
    if (g_isa < 0) g_isa = pick_isa();
    int isa = g_isa;
    if (force_bits) isa = std::min(g_isa, force_bits >= 512 ? 2 : force_bits >= 256 ? 1 : 0);  // never above what the CPU has
    // streaming (non-temporal) stores need their natural alignment: rows that are 16- but not 32-byte aligned (a
    // malloc'ed caller buffer) take the 128-bit path, which still streams; unaligned rows fall back to plain stores
    if ((((uintptr_t)row_out) & 31u) != 0) isa = 0;
    if (isa == 2) expand_avx512(L, rec, row_out);
    else if (isa == 1) expand_avx2(L, rec, row_out);
    else expand_sse2(L, rec, row_out);
}

// ---- worker pool --------------------------------------------------------------------------------------------------
namespace {
// CPUs of every NUMA node, from /sys/devices/system/node/node<k>/cpulist ("0-31,64-95")
std::vector<std::vector<int>> numa_nodes() {
    std::vector<std::vector<int>> nodes;
    for (int k = 0; k < 64; ++k) {
        char path[96];
        snprintf(path, sizeof(path), "/sys/devices/system/node/node%d/cpulist", k);
        FILE *f = fopen(path, "r");
        if (!f) break;
        char buf[4096];
        std::vector<int> cpus;
        if (fgets(buf, sizeof(buf), f)) {
            const char *p = buf;
            while (*p && *p != '\n') {
                char *e;
                long a = strtol(p, &e, 10), b = a;
                if (e == p) break;
                p = e;
                if (*p == '-') {
                    b = strtol(p + 1, &e, 10);
                    p = e;
                }
                for (long c = a; c <= b; ++c) cpus.push_back((int)c);
                if (*p == ',') ++p;
            }
        }
        fclose(f);
        if (!cpus.empty()) nodes.push_back(cpus);
    }
    return nodes;
}
}  // namespace

struct Pool::Impl {
    std::vector<std::thread> th;
    std::mutex mu;
    std::condition_variable cv, done_cv;
    const std::function<void(size_t)> *fn = nullptr;
    size_t n = 0, key0 = 0, pending = 0;
    uint64_t gen = 0;
    bool stop = false, busy = false;
    std::string desc;
    void loop(unsigned me, unsigned nt) {
        uint64_t seen = 0;
        for (;;) {
            const std::function<void(size_t)> *f;
            size_t cnt, k0;
            {
                std::unique_lock<std::mutex> lk(mu);
                cv.wait(lk, [&] { return stop || gen != seen; });
                if (stop) return;
                seen = gen;
                f = fn;
                cnt = n;
                k0 = key0;
            }
            // my items: i with (k0 + i) % nt == me
            size_t first = (me + nt - (k0 % nt)) % nt;
            for (size_t i = first; i < cnt; i += nt) (*f)(i);
            bool last;
            {
                std::lock_guard<std::mutex> lk(mu);
                last = --pending == 0;
            }
            if (last) done_cv.notify_all();
        }
    }
};

Pool &Pool::get(int node_hint) {
    static Pool p(node_hint);
    return p;
}
unsigned Pool::size() const { return (unsigned)p_->th.size(); }
const char *Pool::describe() const { return p_->desc.c_str(); }

Pool::Pool(int node_hint) : p_(new Impl()) {
    unsigned hw = std::max(1u, std::thread::hardware_concurrency());
    // several ranks of one host share its cores and its memory controllers (torchrun sets LOCAL_WORLD_SIZE)
    unsigned ranks = (unsigned)std::max(1, env_int("LOCAL_WORLD_SIZE", 1));
    std::vector<std::vector<int>> nodes = numa_nodes();
    const bool pin = env_int("CW_UNPACK_PIN", 1) != 0 && !nodes.empty();
    std::vector<int> use;  // NUMA nodes the workers live on
    if (pin) {
        if (ranks > 1 && node_hint >= 0 && node_hint < (int)nodes.size()) use.push_back(node_hint);
        else
            for (size_t k = 0; k < nodes.size(); ++k) use.push_back((int)k);
    }
    // streaming stores saturate a host's memory system with a few threads per node; many more threads than that
    // are slower and erratic, so the default stays at half the hardware threads per rank, 4 to 16
    unsigned dflt = std::max(4u, std::min(16u, hw / 2 / ranks));
    unsigned nt = (unsigned)std::max(1, env_int("CW_UNPACK_THREADS", (int)dflt));
    nt = std::min(nt, hw);
    for (unsigned i = 0; i < nt; ++i) {
        p_->th.emplace_back([this, i, nt] { p_->loop(i, nt); });
        if (pin) {
            const std::vector<int> &cpus = nodes[use[i % use.size()]];
            cpu_set_t set;
            CPU_ZERO(&set);
            for (int c : cpus)
                if (c < CPU_SETSIZE) CPU_SET(c, &set);
            pthread_setaffinity_np(p_->th.back().native_handle(), sizeof(set), &set);
        }
    }
    p_->desc = std::to_string(nt) + " threads" +
               (pin ? ", pinned round robin to " + std::to_string(use.size()) + " of " + std::to_string(nodes.size()) + " NUMA nodes" : ", unpinned") +
               ", static item -> thread map, " + expand_isa() + " stores";
}
Pool::~Pool() {
    {
        std::lock_guard<std::mutex> lk(p_->mu);
        p_->stop = true;
    }
    p_->cv.notify_all();
    for (auto &t : p_->th) t.join();
    delete p_;
}

void Pool::parallel_for(size_t n, size_t key0, const std::function<void(size_t)> &fn) {
    if (n == 0) return;
    Impl &I = *p_;
    std::unique_lock<std::mutex> lk(I.mu);
    I.done_cv.wait(lk, [&] { return !I.busy; });  // one parallel_for at a time
    I.busy = true;
    I.fn = &fn;
    I.n = n;
    I.key0 = key0;
    I.pending = I.th.size();
    ++I.gen;
    lk.unlock();
    I.cv.notify_all();
    lk.lock();
    I.done_cv.wait(lk, [&] { return I.pending == 0; });
    I.busy = false;
    I.fn = nullptr;
    lk.unlock();
    I.done_cv.notify_all();
}

}  // namespace cw
