// C ABI (include/circom_b200.h) over the lowering (flatten.cpp), the formats (formats.cpp) and the
// sm_90a kernels (kernels.cuh).  There is no CPU execution path: every compute entry point
// returns CW_ENODEV when no CUDA device is present.
#include <cuda_runtime.h>
#include <dlfcn.h>
#include <emmintrin.h>
#include <nccl.h>

#include <cstdio>
#include <cstdlib>
#include <algorithm>
#include <atomic>
#include <chrono>
#include <condition_variable>
#include <cstring>
#include <functional>
#include <map>
#include <tuple>
#include <memory>
#include <mutex>
#include <thread>
#include <stdexcept>
#include <cerrno>
#include <sys/random.h>
#include <string>
#include <vector>

#include "../../include/circom_b200.h"
#include <cub/device/device_radix_sort.cuh>

#include "kernels.cuh"
#include "msm.cuh"
#include "msm_g2.h"
#include "msm_bls12381.h"
#include "msm_bls12381_g2.h"
#include "groth16.h"
#include "tape_calls.h"
#include "tape.h"
#include "hostpack.h"

using namespace cw;

namespace {

thread_local std::string g_err;
int fail(int code, const std::string &msg) {
    g_err = msg;
    return code;
}
#define CU(call)                                                                                       \
    do {                                                                                               \
        cudaError_t e_ = (call);                                                                       \
        if (e_ != cudaSuccess)                                                                         \
            return fail(CW_ECUDA, std::string(#call) + ": " + cudaGetErrorString(e_));                 \
    } while (0)

// Owners of device memory, pinned host memory, events and streams: the only code that releases them, so that a
// function may return (CU) at any point without leaking what it holds.  Release on the device that is current.
struct DevFree { void operator()(void *p) const { cudaFree(p); } };
struct PinnedFree { void operator()(void *p) const { cudaFreeHost(p); } };
struct EventDestroy { void operator()(cudaEvent_t e) const { cudaEventDestroy(e); } };
struct StreamDestroy { void operator()(cudaStream_t s) const { cudaStreamDestroy(s); } };
template <class T> using DevPtr = std::unique_ptr<T, DevFree>;
template <class T> using PinnedPtr = std::unique_ptr<T, PinnedFree>;
using Event = std::unique_ptr<CUevent_st, EventDestroy>;
using Stream = std::unique_ptr<CUstream_st, StreamDestroy>;

template <class T>
int dev_alloc(DevPtr<T> &dst, size_t bytes) {
    void *p = nullptr;
    CU(cudaMalloc(&p, bytes));
    dst.reset((T *)p);
    return CW_OK;
}
template <class T>
int pinned_alloc(PinnedPtr<T> &dst, size_t bytes) {
    void *p = nullptr;
    CU(cudaMallocHost(&p, bytes));
    dst.reset((T *)p);
    return CW_OK;
}
int make_event(Event &e, unsigned flags = cudaEventDefault) {
    cudaEvent_t h = nullptr;
    CU(cudaEventCreateWithFlags(&h, flags));
    e.reset(h);
    return CW_OK;
}
int make_stream(Stream &s) {
    cudaStream_t h = nullptr;
    CU(cudaStreamCreateWithFlags(&h, cudaStreamNonBlocking));
    s.reset(h);
    return CW_OK;
}
// `bytes` of host memory copied into a new device allocation (at least 16 bytes, so that empty tables get a pointer)
template <class T>
int upload(DevPtr<T> &dst, const void *src, size_t bytes) {
    int rc = dev_alloc(dst, bytes ? bytes : 16);
    if (rc) return rc;
    if (bytes) CU(cudaMemcpy(dst.get(), src, bytes, cudaMemcpyHostToDevice));
    return CW_OK;
}

std::mutex g_dev_mutex;
std::map<int, bool> g_dev_ready;

int ensure_device(int device) {
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess || n == 0) {
        cudaGetLastError();
        return fail(CW_ENODEV, "no CUDA device available (circom_b200 has no CPU execution path)");
    }
    if (device < 0 || device >= n) return fail(CW_EINVAL, "bad device index");
    CU(cudaSetDevice(device));
    std::lock_guard<std::mutex> lk(g_dev_mutex);
    if (!g_dev_ready[device]) {
        FrParams h[N_PRIMES_DEV];
        static_assert(N_PRIMES_DEV == CW_N_PRIMES, "prime tables");
        for (int k = 0; k < N_PRIMES_DEV; ++k) h[k] = make_dev_params(make_field(k));
        CU(cudaMemcpyToSymbol(c_fr, h, sizeof(h)));
        CU(tape_calls_set_params(h, sizeof(h)));
        CU(msm_g2_set_params(h, sizeof(h)));
        CU(msm_bls12381_set_params());
        CU(msm_bls12381_g2_set_params());
        CU(groth16_set_params(h, sizeof(h)));
        g_dev_ready[device] = true;
    }
    return CW_OK;
}

// streaming multiprocessors of the current device: the grid caps of the grid-stride kernels and the tile size
// cw_batch_create picks are counted in SMs
u32 device_sms() {
    int dev = 0, n = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess ||
        n <= 0) {
        cudaGetLastError();
        return 132;   // H100 SXM
    }
    return (u32)n;
}

// Grid of a grid-stride kernel: CTAs of `threads` for `items`, at most `ctas_per_sm` per SM and at least one.  With `rows`
// the kernel strides over that many instances, tiles or vectors in y, where a grid ends at 65,535.
u32 grid_for(uint64_t items, u32 threads, u32 ctas_per_sm) {
    return (u32)std::max<uint64_t>(1, std::min<uint64_t>((items + threads - 1) / threads, (uint64_t)device_sms() * ctas_per_sm));
}
dim3 grid_for(uint64_t items, u32 threads, u32 ctas_per_sm, u32 rows) {
    return dim3(grid_for(items, threads, ctas_per_sm), std::min<u32>(rows, 65535u));
}

struct DevTape {
    DevPtr<uint4> ops;
    DevPtr<u32> items, level_start, level_info;
    bool has_slow = false;
    DevPtr<uint4> heads;  // first tape word of every work item
    DevPtr<uint4> consts;
    DevPtr<u32> input_slot, fn_code, fn_info, call_tab;
    DevPtr<u32> wloc;  // per witness entry: where its value lives (slot id, or OPERAND_BIT | plane position)
    // witness entries outside the bit plane by static size class (slot ids), for the packed device->host transfer
    DevPtr<u32> pk_bit, pk_u64, pk_full;
    TapeDev view;  // what the kernels take (vm_wide is set per run)
};
struct DevR1cs {
    DevPtr<unsigned long long> row_ptr;
    DevPtr<uint4> terms;  // per term {location, dictionary index, kind word, absorbed boolean row}
    DevPtr<uint4> dictM;
    DevPtr<u32> perm, bool_loc, bool_row;
    DevPtr<u32> perm_small;   // rows small by shape: decided over the integers (r1cs_small.h)
    DevPtr<uint2> sgroups, srecs;   // ... from a term list of their own
    DevPtr<u32> sbrow;
    u32 n_general = 0, n_bool = 0, n_small = 0;
    u32 mean_row_terms = 0;  // compiled terms per general row
    uint64_t n_terms = 0;
    R1csDev general, integer;   // what the kernels take: the general rows, the integer rows
    R1csSmallDev integer_recs;
};

int env_int(const char *name, int dflt) {
    const char *s = getenv(name);
    return s && *s ? atoi(s) : dflt;
}

}  // namespace

// Packed-transfer layout from the classes the witness values were SEEN to have (narrower than the proven ones; kernels.cuh:
// witness_observe_kernel), with the device copies of its location lists.  One per circuit and device, replaced (never
// edited) when a batch shows a wider value; transfers hold a reference while they use it.
struct NarrowPack {
    PackLayout L;
    std::vector<uint8_t> cls;
    DevPtr<u32> pk_bit, pk_u64, pk_full;
};

static std::atomic<uint64_t> g_circuit_serial{0};

struct cw_circuit {
    const uint64_t serial = ++g_circuit_serial;   // process-wide identity of the handle (never 0): the R1CS layout key
    Tape tape;
    mutable std::mutex mu;
    mutable std::mutex narrow_mu;   // serialises the (rare) observation passes
    mutable std::map<int, std::shared_ptr<NarrowPack>> narrow;   // guarded by mu
    mutable std::map<int, DevTape> dev;
    mutable PackLayout pack;
    mutable bool pack_ready = false;
    const PackLayout &pack_layout() const {
        std::lock_guard<std::mutex> lk(mu);
        if (!pack_ready) {
            build_pack_layout(tape, pack);
            pack_ready = true;
        }
        return pack;
    }
};

struct R1csKey {
    int device;
    uint64_t layout;  // serial of the circuit whose value layout the CSR reads; 0: dense witness rows (location = wire id)
    bool operator<(const R1csKey &o) const { return device != o.device ? device < o.device : layout < o.layout; }
};
struct cw_r1cs {
    R1csData data;
    FieldParams F;
    std::mutex mu;
    std::map<R1csKey, DevR1cs> dev;
    std::unique_ptr<cw_r1cs> eval_twin;  // the same constraints compiled without boolean-row special cases (cw_r1cs_eval_batch)
    std::unique_ptr<cw_r1cs> qap_twin;   // ... plus the rows a_{m+j} = w_j, j <= nPublic (cw_r1cs_quotient_*)
    uint64_t digest = 0;                 // content hash of the constraints (r1cs_digest; 0: not computed yet)
    bool no_bool_rows = false;
};

struct cw_batch {
    const cw_circuit *c = nullptr;
    int device = 0;
    u32 batch = 0, batch_padded = 0, bt_log2 = 0, threads = 256;
    Stream stream;   // (declared first: released last)
    DevPtr<uint4> slots, inputs_d, witness_d;
    DevPtr<u32> plane;
    DevPtr<u32> first_assert_d;
    DevPtr<int> err_d;
    DevPtr<unsigned long long> fb_d;  // per-instance result of the R1CS check
    DevPtr<u32> r1cs_wide_d;          // bitmap of the integer rows handed to the general kernel (launch_r1cs)
    u32 r1cs_wide_rows = 0;
    const DevTape *dt = nullptr;      // the circuit's cache entry for this device
    std::vector<uint64_t> host_inputs;  // [batch][n_inputs][4]
    std::vector<uint8_t> assigned;      // [batch][n_inputs]
    std::vector<u32> remaining;         // [batch]
    bool host_inputs_dirty = false;
    bool inputs_on_device = false;
    bool ran = false;
    bool dense_valid = false;  // witness_d holds the dense rows of the current run
    // packed transfer: two staging buffers (device + pinned host) so that the pack kernel and the copy of one
    // chunk overlap the host-side expansion of the previous one
    DevPtr<u32> packed_d[2];
    PinnedPtr<u32> packed_h[2];
    size_t packed_cap = 0;  // instances per staging buffer
    DevPtr<uint4> dense_chunk_d;
    size_t dense_chunk_cap = 0;
    DevPtr<int> pack_flag_d;  // set by the pack kernel when a value exceeds its class
    Event pack_ev[2];
    uint64_t last_d2h_bytes = 0;
    Event ev[3];
    std::thread async_th;  // cw_batch_get_witness_async
    int async_rc = 0;
    std::string async_err;
    bool async_active = false;
    bool identity_layout() const {  // witness row i = the first n_witness slots of instance i's slot store
        const Tape &t = c->tape;
        return bt_log2 == 0 && t.n_bitwords == 0 && t.n_resident == t.n_witness;
    }
    StoreDev store() const {
        StoreDev S;
        S.slots = slots.get();
        S.plane = plane.get();
        S.n_slots = c->tape.n_slots;
        S.n_bitwords = c->tape.n_bitwords;
        S.bt_log2 = bt_log2;
        S.batch = batch;
        return S;
    }
};

// `count` dense witness rows `stride_elems` elements apart, as a value store (one instance per tile, no bit plane)
static StoreDev dense_store(const void *rows, uint64_t stride_elems, u32 count) {
    StoreDev S;
    S.slots = (const uint4 *)rows;
    S.plane = nullptr;
    S.n_slots = (u32)stride_elems;
    S.n_bitwords = 0;
    S.bt_log2 = 0;
    S.batch = count;
    return S;
}

static int get_dev_tape(const cw_circuit *c, int device, const DevTape *&out) {
    const PackLayout &L = c->pack_layout();
    std::lock_guard<std::mutex> lk(c->mu);
    auto it = c->dev.find(device);
    if (it != c->dev.end()) {
        out = &it->second;
        return CW_OK;
    }
    const Tape &t = c->tape;
    DevTape d;
    int rc;
    if ((rc = upload(d.ops, t.ops.data(), t.ops.size() * 4))) return rc;
    if ((rc = upload(d.items, t.items.data(), t.items.size() * 4))) return rc;
    {
        std::vector<uint32_t> heads(t.n_items() * 4);
        for (size_t k = 0; k < t.n_items(); ++k) memcpy(&heads[k * 4], &t.ops[(size_t)t.items[k] * 4], 16);
        if ((rc = upload(d.heads, heads.data(), heads.size() * 4))) return rc;
    }
    if ((rc = upload(d.level_start, t.level_start.data(), t.level_start.size() * 4))) return rc;
    {
        // per level: how many calls close it (the lowering sorts the items of a level by opcode, CALL is the largest: the
        // kernel runs them after the other items) and whether it has INV / POW items (run in a pass of their own)
        std::vector<uint32_t> info(t.n_levels(), 0);
        for (size_t l = 0; l < t.n_levels(); ++l) {
            bool tail = true;
            for (uint32_t k = t.level_start[l + 1]; k-- > t.level_start[l];) {
                const uint32_t opc = t.ops[(size_t)t.items[k] * 4] & 0xFFu;
                const bool single = t.items[k + 1] - t.items[k] == 1;
                const bool is_call = opc == OP_CALL && single;
                if (opc == OP_CALL && !(single && tail)) return fail(CW_ESTATE, "internal: a call is not at the end of its level");
                if (is_call) ++info[l];
                else tail = false;
                for (uint32_t w = t.items[k]; w < t.items[k + 1]; ++w) {
                    const uint32_t o = t.ops[(size_t)w * 4] & 0xFFu;
                    if (o == OP_INV || o == OP_POW) {
                        if (!single) return fail(CW_ESTATE, "internal: a fused work item contains INV / POW");
                        info[l] |= 0x80000000u;
                        d.has_slow = true;
                    }
                }
            }
        }
        if ((rc = upload(d.level_info, info.data(), info.size() * 4))) return rc;
    }
    if ((rc = upload(d.consts, t.consts.data(), t.consts.size() * 32))) return rc;
    if ((rc = upload(d.input_slot, t.input_slot.data(), t.input_slot.size() * 4))) return rc;
    if ((rc = upload(d.fn_code, t.fn_code.data(), t.fn_code.size() * 4))) return rc;
    if ((rc = upload(d.fn_info, t.fn_info.data(), t.fn_info.size() * 4))) return rc;
    if ((rc = upload(d.call_tab, t.call_tab.data(), t.call_tab.size() * 4))) return rc;
    if ((rc = upload(d.wloc, t.witness_slot.data(), t.witness_slot.size() * 4))) return rc;
    if ((rc = upload(d.pk_bit, L.bit_loc.data(), L.bit_loc.size() * 4))) return rc;
    if ((rc = upload(d.pk_u64, L.u64_loc.data(), L.u64_loc.size() * 4))) return rc;
    if ((rc = upload(d.pk_full, L.full_loc.data(), L.full_loc.size() * 4))) return rc;
    TapeDev &tp = d.view;
    tp.ops = d.ops.get();
    tp.items = d.items.get();
    tp.heads = d.heads.get();
    tp.level_start = d.level_start.get();
    tp.level_info = d.level_info.get();
    tp.has_slow = d.has_slow ? 1u : 0u;
    tp.consts = d.consts.get();
    tp.n_levels = (u32)t.n_levels();
    tp.n_slots = t.n_slots;
    tp.input_slot = d.input_slot.get();
    tp.fn_code = d.fn_code.get();
    tp.fn_info = d.fn_info.get();
    tp.call_tab = d.call_tab.get();
    tp.n_inputs = (u32)t.n_inputs;
    tp.n_bitwords = t.n_bitwords;
    tp.prime = (u32)t.F.prime_id;
    tp.vm_wide = 0;
    out = &c->dev.emplace(device, std::move(d)).first->second;
    return CW_OK;
}

// the build of the interpreter a run of b lands on (tape_calls.h: select_tape_build)
static int batch_tape_build(const cw_batch *b, TapeBuild &k) {
    const Tape &t = b->c->tape;
    if (!select_tape_build(t.F.prime_id, !t.call_tab.empty(), t.n_bitwords != 0, t.n_items() != t.n_tape_ops(), b->bt_log2, k))
        return fail(CW_ESTATE, "CW_FLAG_FUSE is available for bn128 and bls12381");
    return CW_OK;
}

// the builds without the function machine are compiled here, the others in tape_calls.cu
static int launch_tape(const TapeBuild &k, const TapeLaunch &a) {
    const bool found = k.calls ? launch_tape_calls(k, a) : with_prime(k.prime, [&](auto pr) {
        constexpr int PR = decltype(pr)::value;
        if constexpr (PR >= 0)
            return launch_tape_k<PR, false, true, 5, true>(k, a) || launch_tape_k<PR, false, true, -1, true>(k, a) ||
                   launch_tape_k<PR, false, true, 0, false>(k, a) || launch_tape_k<PR, false, true, 5, false>(k, a) ||
                   launch_tape_k<PR, false, true, -1, false>(k, a) || launch_tape_k<PR, false, false, 0, false>(k, a) ||
                   launch_tape_k<PR, false, false, -1, false>(k, a);
        else
            return launch_tape_k<-1, false, true, -1, false>(k, a);
    });
    return found ? CW_OK : fail(CW_ESTATE, "internal: the library does not contain the interpreter build of this run");
}

extern "C" {

int cw_version(void) { return 100; }
const char *cw_last_error(void) { return g_err.c_str(); }
int cw_device_count(void) {
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess) {
        cudaGetLastError();
        return 0;
    }
    return n;
}

int cw_circuit_load_mem(const void *data, size_t len, uint32_t flags, cw_circuit **out) {
    if (!data || !out) return fail(CW_EINVAL, "null argument");
    auto c = std::make_unique<cw_circuit>();
    try {
        lower_circuit((const uint8_t *)data, len, flags, c->tape);
    } catch (const std::exception &e) {
        return fail(CW_EFORMAT, e.what());
    }
    *out = c.release();
    return CW_OK;
}

int cw_circuit_load(const char *path, uint32_t flags, cw_circuit **out) {
    if (!path || !out) return fail(CW_EINVAL, "null argument");
    FILE *f = fopen(path, "rb");
    if (!f) return fail(CW_EIO, std::string("cannot open ") + path);
    fseek(f, 0, SEEK_END);
    long sz = ftell(f);
    fseek(f, 0, SEEK_SET);
    std::vector<uint8_t> buf(sz);
    size_t rd = sz ? fread(buf.data(), 1, sz, f) : 0;
    fclose(f);
    if ((long)rd != sz) return fail(CW_EIO, "short read");
    return cw_circuit_load_mem(buf.data(), buf.size(), flags, out);
}

void cw_circuit_destroy(cw_circuit *c) {
    if (!c) return;
    for (auto it = c->dev.begin(); it != c->dev.end(); it = c->dev.erase(it)) {
        cudaSetDevice(it->first);
        c->narrow.erase(it->first);
    }
    delete c;
}

int cw_circuit_stats(const cw_circuit *c, cw_stats *o) {
    if (!c || !o) return fail(CW_EINVAL, "null argument");
    const Tape &t = c->tape;
    memset(o, 0, sizeof(*o));
    o->n_signals = t.n_signals;
    o->n_witness = t.n_witness;
    o->n_inputs = t.n_inputs;
    o->n_outputs = t.n_outputs;
    o->n_components = t.n_components;
    o->n_constants = t.consts.size();
    o->n_ir_ops = t.n_ir_ops;
    o->n_tape_ops = t.n_tape_ops();
    o->n_slots = t.n_slots;
    o->n_levels = t.n_levels();
    o->n_constraints = t.r1cs.n_constraints;
    o->n_nnz = t.r1cs.col.size();
    o->n_mul_ops = t.n_mul_ops;
    o->n_conv_ops = t.n_conv_ops;
    o->max_level_width = t.max_level_width;
    o->n_slot_operands = t.n_slot_operands;
    o->n_bitwords = t.n_bitwords;
    o->n_resident_slots = t.n_resident;
    o->n_values = t.n_values;
    o->n_items = t.n_items();
    o->n_stored = t.n_stored;
    return CW_OK;
}

int cw_circuit_prime(const cw_circuit *c, int *prime_id, uint64_t q[4]) {
    if (!c) return fail(CW_EINVAL, "null argument");
    if (prime_id) *prime_id = c->tape.F.prime_id;
    if (q) memcpy(q, c->tape.F.q.v, 32);
    return CW_OK;
}

uint32_t cw_get_main_input_signal_start(const cw_circuit *c) { return (uint32_t)c->tape.n_outputs + 1; }
uint32_t cw_get_main_input_signal_no(const cw_circuit *c) { return (uint32_t)c->tape.n_inputs; }
uint32_t cw_get_total_signal_no(const cw_circuit *c) { return (uint32_t)c->tape.n_signals; }
uint32_t cw_get_number_of_components(const cw_circuit *c) { return (uint32_t)c->tape.n_components; }
uint32_t cw_get_size_of_input_hashmap(const cw_circuit *c) { return (uint32_t)c->tape.hashmap.size(); }
uint32_t cw_get_size_of_witness(const cw_circuit *c) { return (uint32_t)c->tape.n_witness; }
uint32_t cw_get_size_of_constants(const cw_circuit *c) { return (uint32_t)c->tape.consts.size(); }

uint64_t cw_fnv1a(const char *name) { return fnv1a(name, strlen(name)); }

// getInputSignalHashPosition (calcwit.cpp:51-69)
static int hash_pos(const Tape &t, uint64_t h, size_t *pos) {
    size_t n = t.hashmap.size();
    size_t p = (size_t)(h % n);
    if (t.hashmap[p].hash != h || t.hashmap[p].signalid == 0) {
        size_t ini = p;
        p = (p + 1) % n;
        while (p != ini) {
            if (t.hashmap[p].hash == h && t.hashmap[p].signalid != 0) {
                *pos = p;
                return CW_OK;
            }
            if (t.hashmap[p].signalid == 0) return fail(CW_ENOTFOUND, "Signal not found");
            p = (p + 1) % n;
        }
        return fail(CW_ENOTFOUND, "Signals not found");
    }
    *pos = p;
    return CW_OK;
}

int cw_get_input_signal_size(const cw_circuit *c, uint64_t h, uint64_t *size) {
    size_t p;
    int rc = hash_pos(c->tape, h, &p);
    if (rc) return rc;
    *size = c->tape.hashmap[p].signalsize;
    return CW_OK;
}
int cw_get_input_signal_id(const cw_circuit *c, uint64_t h, uint64_t *id) {
    size_t p;
    int rc = hash_pos(c->tape, h, &p);
    if (rc) return rc;
    *id = c->tape.hashmap[p].signalid;
    return CW_OK;
}

int cw_circuit_tape_items(const cw_circuit *c, uint32_t *items) {
    if (!c || !items) return fail(CW_EINVAL, "null argument");
    memcpy(items, c->tape.items.data(), c->tape.items.size() * 4);
    return CW_OK;
}

int cw_circuit_tape(const cw_circuit *c, uint32_t *ops, uint32_t *level_start, uint32_t *witness_slot) {
    const Tape &t = c->tape;
    if (ops) memcpy(ops, t.ops.data(), t.ops.size() * 4);
    if (level_start) memcpy(level_start, t.level_start.data(), t.level_start.size() * 4);
    if (witness_slot) memcpy(witness_slot, t.witness_slot.data(), t.witness_slot.size() * 4);
    return CW_OK;
}

int cw_circuit_slot_census(const cw_circuit *c, uint64_t out[4]) {
    if (!c || !out) return fail(CW_EINVAL, "null argument");
    memcpy(out, c->tape.slot_census, sizeof(c->tape.slot_census));
    return CW_OK;
}

int cw_circuit_width_census(const cw_circuit *c, uint64_t out[256]) {
    if (!c || !out) return fail(CW_EINVAL, "null argument");
    memcpy(out, c->tape.width_census, sizeof(c->tape.width_census));
    return CW_OK;
}

int cw_circuit_witness2signal(const cw_circuit *c, uint64_t *out) {
    if (!c || !out) return fail(CW_EINVAL, "null argument");
    memcpy(out, c->tape.witness2signal.data(), c->tape.witness2signal.size() * 8);
    return CW_OK;
}

int cw_circuit_write_dat(const cw_circuit *c, const char *path) {
    try {
        write_dat(c->tape, path);
    } catch (const std::exception &e) {
        return fail(CW_EIO, e.what());
    }
    return CW_OK;
}

int cw_circuit_functions(const cw_circuit *c, uint32_t *n, uint32_t *info) {
    if (!c || !n) return fail(CW_EINVAL, "null argument");
    *n = (uint32_t)(c->tape.fn_info.size() / 4);
    if (info) memcpy(info, c->tape.fn_info.data(), c->tape.fn_info.size() * 4);
    return CW_OK;
}

int cw_circuit_write_sym(const cw_circuit *c, const char *path) {
    if (!c || !path) return fail(CW_EINVAL, "null argument");
    if (c->tape.sym.empty()) return fail(CW_ESTATE, "the circuit description carries no symbols section");
    try {
        write_sym(c->tape, path);
    } catch (const std::exception &e) {
        return fail(CW_EIO, e.what());
    }
    return CW_OK;
}

// ---- batch ------------------------------------------------------------------------------------
int cw_batch_create(const cw_circuit *c, uint32_t batch, int device, cw_batch **out) {
    if (!c || !out || batch == 0) return fail(CW_EINVAL, "bad argument");
    if (c->tape.flags & CW_FLAG_HOST_ONLY) return fail(CW_ESTATE, "circuit was loaded with CW_FLAG_HOST_ONLY");
    int rc = ensure_device(device);
    if (rc) return rc;
    const Tape &t = c->tape;
    auto b = std::make_unique<cw_batch>();
    b->c = c;
    b->device = device;
    b->batch = batch;
    // Tile size (instances side by side in the slot store).  Lanes along instances (32-instance tiles: a warp is one
    // op, every access coalesced, no divergence) need enough tiles to fill the GPU with CTAs; below that, lanes run
    // along the ops of a level (one-instance tiles).
    int bt = env_int("CW_BT_LOG2", -1);
    const uint64_t avg_w = t.n_levels() ? t.n_items() / t.n_levels() + 1 : 1;
    const u32 sms = device_sms();
    if (bt < 0) {
        bt = 0;
        if (batch >= 32u * sms * 2u) bt = 5;   // (also with function calls: the 32 lanes run the same function body)
        else if (t.call_tab.empty())
            while (bt < 5 && (avg_w << bt) < 64 && (batch >> (bt + 1)) >= 2u * sms) ++bt;  // very narrow tapes (Poseidon)
    }
    if (bt > 5) bt = 5;
    b->bt_log2 = (u32)bt;
    u32 btn = 1u << bt;
    b->batch_padded = (batch + btn - 1) / btn * btn;
    int th = env_int("CW_THREADS", 0);
    if (th <= 0) {
        // enough threads for a typical level: average width x tile, clamped to [64, 512]
        uint64_t avg = avg_w * btn;
        th = 64;
        while (th < 512 && (uint64_t)th < avg) th <<= 1;
        // many tiles per SM hide latency better than wide CTAs: keep <= ~1024 resident threads per SM
        u32 tiles = b->batch_padded >> bt;
        u32 per_sm = (tiles + sms - 1) / sms;
        while (th > 64 && (u32)th * per_sm > 1024) th >>= 1;
        if (tiles < sms) th = CW_TAPE_LB;  // fewer tiles than SMs: the widest CTA (wide levels finish in one pass)
    }
    th = (th + 31) / 32 * 32;
    if (th > CW_TAPE_LB) th = CW_TAPE_LB;
    b->threads = (u32)th;
    size_t slot_bytes = (size_t)b->batch_padded * t.n_slots * 32;
    size_t plane_bytes = (size_t)b->batch_padded * t.n_bitwords * 4;
    size_t free_b = 0, total_b = 0;
    cudaMemGetInfo(&free_b, &total_b);
    size_t need = slot_bytes + plane_bytes + (size_t)batch * t.n_inputs * 32 + (64u << 20);
    if (need > free_b)
        return fail(CW_ECUDA, "batch needs " + std::to_string(need >> 20) + " MiB of device memory, " +
                                  std::to_string(free_b >> 20) + " MiB free");
    if ((rc = get_dev_tape(c, device, b->dt))) return rc;
    if ((rc = make_stream(b->stream))) return rc;
    if ((rc = dev_alloc(b->slots, slot_bytes))) return rc;
    if ((rc = dev_alloc(b->plane, std::max<size_t>(plane_bytes, 16)))) return rc;
    if ((rc = dev_alloc(b->inputs_d, std::max<size_t>((size_t)batch * t.n_inputs * 32, 32)))) return rc;
    if ((rc = dev_alloc(b->first_assert_d, (size_t)batch * 4))) return rc;
    if ((rc = dev_alloc(b->err_d, (size_t)batch * 4))) return rc;
    if ((rc = dev_alloc(b->fb_d, (size_t)batch * 8))) return rc;
    if ((rc = dev_alloc(b->pack_flag_d, 4))) return rc;
    for (auto &e : b->ev)
        if ((rc = make_event(e))) return rc;
    for (auto &e : b->pack_ev)
        if ((rc = make_event(e, cudaEventDisableTiming))) return rc;
    b->host_inputs.assign((size_t)batch * t.n_inputs * 4, 0);
    b->assigned.assign((size_t)batch * t.n_inputs, 0);
    b->remaining.assign(batch, (u32)t.n_inputs);
    *out = b.release();
    return CW_OK;
}

static void join_async(cw_batch *b) {
    if (b->async_th.joinable()) b->async_th.join();
    b->async_active = false;
}

void cw_batch_destroy(cw_batch *b) {
    if (!b) return;
    join_async(b);   // (the helper thread uses the members)
    cudaSetDevice(b->device);
    delete b;
}

int cw_batch_layout(const cw_batch *b, uint32_t *bt_log2, uint32_t *threads, uint64_t *bytes_per_instance) {
    if (!b) return fail(CW_EINVAL, "null argument");
    if (bt_log2) *bt_log2 = b->bt_log2;
    if (threads) *threads = b->threads;
    if (bytes_per_instance) *bytes_per_instance = (uint64_t)b->c->tape.n_slots * 32 + (uint64_t)b->c->tape.n_bitwords * 4;
    return CW_OK;
}

int cw_batch_tape_build(const cw_batch *b, int32_t out[5]) {
    if (!b || !out) return fail(CW_EINVAL, "null argument");
    TapeBuild k;
    int rc = batch_tape_build(b, k);
    if (rc) return rc;
    out[0] = k.prime;
    out[1] = k.calls;
    out[2] = k.bp;
    out[3] = k.bt;
    out[4] = k.fused;
    return CW_OK;
}

int cw_batch_set_input(cw_batch *b, uint32_t inst, uint64_t h, uint32_t idx, const uint64_t limbs[4]) {
    if (!b || inst >= b->batch) return fail(CW_EINVAL, "bad instance");
    const Tape &t = b->c->tape;
    if (b->remaining[inst] == 0) return fail(CW_ESTATE, "No more signals to be assigned");
    size_t p;
    int rc = hash_pos(t, h, &p);
    if (rc) return rc;
    if (idx >= t.hashmap[p].signalsize) return fail(CW_EINVAL, "Input signal array access exceeds the size");
    uint64_t si = t.hashmap[p].signalid + idx;
    uint64_t k = si - (t.n_outputs + 1);
    if (si < t.n_outputs + 1 || k >= t.n_inputs) return fail(CW_EINVAL, "input signal outside the main inputs");
    if (b->assigned[(size_t)inst * t.n_inputs + k]) return fail(CW_ESTATE, "Signal assigned twice: " + std::to_string(si));
    U256 v;
    memcpy(v.v, limbs, 32);
    if (!(v < t.F.q)) return fail(CW_EINVAL, "input value not reduced modulo the field prime");
    memcpy(&b->host_inputs[((size_t)inst * t.n_inputs + k) * 4], limbs, 32);
    b->assigned[(size_t)inst * t.n_inputs + k] = 1;
    b->remaining[inst]--;
    b->host_inputs_dirty = true;
    return CW_OK;
}

int cw_batch_remaining_inputs(const cw_batch *b, uint32_t inst, uint32_t *rem) {
    if (!b || inst >= b->batch) return fail(CW_EINVAL, "bad instance");
    *rem = b->remaining[inst];
    return CW_OK;
}

int cw_batch_set_inputs(cw_batch *b, const uint64_t *inputs, int is_device_ptr) {
    if (!b || !inputs) return fail(CW_EINVAL, "null argument");
    if (b->async_active) return fail(CW_ESTATE, "a witness transfer of this batch is in flight (cw_batch_get_witness_wait)");
    const Tape &t = b->c->tape;
    CU(cudaSetDevice(b->device));
    size_t bytes = (size_t)b->batch * t.n_inputs * 32;
    CU(cudaMemcpyAsync(b->inputs_d.get(), inputs, bytes, is_device_ptr ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice,
                       b->stream.get()));
    std::fill(b->remaining.begin(), b->remaining.end(), 0u);
    b->host_inputs_dirty = false;
    b->inputs_on_device = true;
    return CW_OK;
}

int cw_batch_run(cw_batch *b) {
    if (!b) return fail(CW_EINVAL, "null argument");
    if (b->async_active) return fail(CW_ESTATE, "a witness transfer of this batch is in flight (cw_batch_get_witness_wait)");
    const Tape &t = b->c->tape;
    CU(cudaSetDevice(b->device));
    if (b->host_inputs_dirty || !b->inputs_on_device) {
        for (u32 i = 0; i < b->batch; ++i)
            if (b->remaining[i])
                return fail(CW_ESTATE, "Not all inputs have been set. Only " +
                                           std::to_string(t.n_inputs - b->remaining[i]) + " out of " +
                                           std::to_string(t.n_inputs) + " (instance " + std::to_string(i) + ")");
        CU(cudaMemcpyAsync(b->inputs_d.get(), b->host_inputs.data(), b->host_inputs.size() * 8, cudaMemcpyHostToDevice,
                           b->stream.get()));
        b->host_inputs_dirty = false;
        b->inputs_on_device = true;
    }
    TapeDev tp = b->dt->view;
    // the 128-bit register machine computes over the integers and gives up when a value leaves 128 bits: right only for a
    // prime above 2^128 (every 256-bit one); goldilocks calls run on the full-width machine
    tp.vm_wide = (env_int("CW_VM_WIDE", 0) || t.F.qbits <= 128) ? 1u : 0u;
    CU(cudaMemsetAsync(b->first_assert_d.get(), 0xFF, (size_t)b->batch * 4, b->stream.get()));
    CU(cudaMemsetAsync(b->err_d.get(), 0, (size_t)b->batch * 4, b->stream.get()));
    CU(cudaEventRecord(b->ev[0].get(), b->stream.get()));
    stage_inputs_kernel<<<grid_for((uint64_t)b->batch_padded * (t.n_inputs + 1), 256, 8), 256, 0, b->stream.get()>>>(
        tp, b->inputs_d.get(), b->slots.get(), b->batch, b->batch_padded, b->bt_log2);
    if (tp.n_levels) {
        TapeBuild k;
        int rc = batch_tape_build(b, k);
        if (rc) return rc;
        const u32 th = k.calls ? std::min<u32>(b->threads, 256u) : b->threads;  // the interpreter build has a large frame
        const TapeLaunch a{tp, b->slots.get(), b->plane.get(), b->bt_log2, b->first_assert_d.get(), b->err_d.get(), b->batch,
                           b->batch_padded >> b->bt_log2, th, b->stream.get()};
        if ((rc = launch_tape(k, a))) return rc;
    }
    CU(cudaEventRecord(b->ev[1].get(), b->stream.get()));
    b->dense_valid = false;
    CU(cudaEventRecord(b->ev[2].get(), b->stream.get()));
    CU(cudaGetLastError());
    b->ran = true;
    return CW_OK;
}

int cw_batch_sync(cw_batch *b) {
    if (!b) return fail(CW_EINVAL, "null argument");
    CU(cudaSetDevice(b->device));
    CU(cudaStreamSynchronize(b->stream.get()));
    return CW_OK;
}

int cw_batch_status(cw_batch *b, int32_t *status) {
    if (!b || !status) return fail(CW_EINVAL, "null argument");
    if (!b->ran) return fail(CW_ESTATE, "batch has not been run");
    CU(cudaSetDevice(b->device));
    std::vector<u32> fa(b->batch);
    std::vector<int> er(b->batch);
    CU(cudaMemcpyAsync(fa.data(), b->first_assert_d.get(), (size_t)b->batch * 4, cudaMemcpyDeviceToHost, b->stream.get()));
    CU(cudaMemcpyAsync(er.data(), b->err_d.get(), (size_t)b->batch * 4, cudaMemcpyDeviceToHost, b->stream.get()));
    CU(cudaStreamSynchronize(b->stream.get()));
    for (u32 i = 0; i < b->batch; ++i) {
        if (er[i]) status[i] = -1;  // division by zero: the reference process aborts inside GMP
        else status[i] = fa[i] == 0xFFFFFFFFu ? 0 : (int32_t)(fa[i] + 1);
    }
    return CW_OK;
}

// dense witness rows of instances [first, first + count) into `dst` (device, 32-byte aligned), on the batch stream
static int expand_rows(cw_batch *b, u32 first, u32 count, uint4 *dst) {
    const Tape &t = b->c->tape;
    if (count == 0) return CW_OK;
    witness_expand_kernel<<<grid_for(t.n_witness, 256, 4, count), 256, 0, b->stream.get()>>>(b->store(), b->dt->wloc.get(),
                                                                                             (u32)t.n_witness, first, count, dst);
    CU(cudaGetLastError());
    return CW_OK;
}

// contiguous [batch][n_witness] copy in device memory, for callers that want the reference's layout on the device
static int dense_witness(cw_batch *b) {
    if (b->dense_valid) return CW_OK;
    const Tape &t = b->c->tape;
    int rc;
    if (!b->witness_d) {
        size_t bytes = (size_t)b->batch * t.n_witness * 32, free_b = 0, total_b = 0;
        cudaMemGetInfo(&free_b, &total_b);
        if (bytes + (64u << 20) > free_b)
            return fail(CW_ECUDA, "dense witness rows of the whole batch need " + std::to_string(bytes >> 20) +
                                      " MiB of device memory (" + std::to_string(free_b >> 20) +
                                      " MiB free): use cw_batch_expand_witness on a range of instances");
        if ((rc = dev_alloc(b->witness_d, bytes))) return rc;
    }
    rc = expand_rows(b, 0, b->batch, b->witness_d.get());
    if (rc) return rc;
    b->dense_valid = true;
    return CW_OK;
}

int cw_batch_expand_witness(cw_batch *b, uint32_t first, uint32_t count, uint64_t *dst_device) {
    if (!b || !dst_device || (uint64_t)first + count > b->batch) return fail(CW_EINVAL, "bad argument");
    if (!b->ran) return fail(CW_ESTATE, "batch has not been run");
    if ((uintptr_t)dst_device & 31u) return fail(CW_EINVAL, "destination must be 32-byte aligned");
    CU(cudaSetDevice(b->device));
    return expand_rows(b, first, count, (uint4 *)dst_device);
}

// NUMA node the GPU hangs off (/sys/bus/pci/devices/<bus id>/numa_node), -1 if unknown
static int device_numa_node(int device) {
    char id[32] = {0};
    if (cudaDeviceGetPCIBusId(id, sizeof(id), device) != cudaSuccess) return -1;
    for (char *p = id; *p; ++p) *p = (char)tolower(*p);
    std::string path = std::string("/sys/bus/pci/devices/") + id + "/numa_node";
    FILE *f = fopen(path.c_str(), "r");
    if (!f) return -1;
    int node = -1;
    if (fscanf(f, "%d", &node) != 1) node = -1;
    fclose(f);
    return node;
}

static size_t pack_chunk_instances(const cw_batch *b, const PackLayout &L) {
    size_t mb = (size_t)std::max(8, env_int("CW_PACK_CHUNK_MB", 96));
    size_t n = std::max<size_t>(1, (mb << 20) / (L.words * 4));
    return std::min<size_t>(n, b->batch);
}

static int ensure_pack_buffers(cw_batch *b, const PackLayout &L) {
    if (b->packed_cap) return CW_OK;
    size_t n = pack_chunk_instances(b, L);
    int rc;
    for (int k = 0; k < 2; ++k) {
        if ((rc = dev_alloc(b->packed_d[k], n * L.words * 4))) return rc;
        if ((rc = pinned_alloc(b->packed_h[k], n * L.words * 4))) return rc;
    }
    b->packed_cap = n;
    return CW_OK;
}

// packed records of instances [first, first + count) into `dst_d` (device), on the batch stream; np: the layout of observed
// classes (else the proven one, whose location lists are part of the device tape)
static int pack_rows(cw_batch *b, const PackLayout &L, u32 first, u32 count, u32 *dst_d, const NarrowPack *np = nullptr) {
    const size_t items = L.n_plane_words + L.n_bit_words + L.u64_loc.size() + L.full_loc.size();
    witness_pack_kernel<<<grid_for(items, 256, 4, count), 256, 0, b->stream.get()>>>(
        b->store(), (np ? np->pk_bit : b->dt->pk_bit).get(), (u32)L.bit_loc.size(), (np ? np->pk_u64 : b->dt->pk_u64).get(),
        (u32)L.u64_loc.size(), (np ? np->pk_full : b->dt->pk_full).get(), (u32)L.full_loc.size(), dst_d, L.words, first, count,
        b->pack_flag_d.get());
    CU(cudaGetLastError());
    return CW_OK;
}

// Looks at the values of a finished batch and (re)builds the circuit's layout of observed classes for the batch's device:
// class = max(what earlier batches showed, what this one shows), never wider than the proven class.
static int observe_classes(cw_batch *b, std::shared_ptr<NarrowPack> prev, std::shared_ptr<NarrowPack> &out) {
    const cw_circuit *c = b->c;
    const Tape &t = c->tape;
    const size_t W = t.n_witness;
    std::lock_guard<std::mutex> guard(c->narrow_mu);
    {   // another transfer may have observed meanwhile: start from the newest
        std::lock_guard<std::mutex> lk(c->mu);
        auto it = c->narrow.find(b->device);
        if (it != c->narrow.end() && it->second != prev) prev = it->second;
    }
    // the entries worth looking at: outside the bit plane, proven class above "bit"
    std::vector<u32> loc, wit;
    for (size_t i = 0; i < W; ++i)
        if (!(t.witness_slot[i] & OPERAND_BIT) && t.wit_class[i] > 0) {
            loc.push_back(t.witness_slot[i]);
            wit.push_back((u32)i);
        }
    auto np = std::make_shared<NarrowPack>();
    np->cls.assign(t.wit_class.begin(), t.wit_class.end());
    if (!loc.empty()) {
        std::vector<u32> cls(loc.size(), 0);
        if (prev)
            for (size_t k = 0; k < loc.size(); ++k) cls[k] = prev->cls[wit[k]];
        DevPtr<u32> loc_d, cls_d;
        int rc;
        if ((rc = upload(loc_d, loc.data(), loc.size() * 4))) return rc;
        if ((rc = upload(cls_d, cls.data(), cls.size() * 4))) return rc;
        const u32 n_tiles = (b->batch + (1u << b->bt_log2) - 1) >> b->bt_log2;
        const uint64_t items = (uint64_t)loc.size() << b->bt_log2;
        witness_observe_kernel<<<grid_for(items, 256, 8, n_tiles), 256, 0, b->stream.get()>>>(b->store(), loc_d.get(),
                                                                                              (u32)loc.size(), cls_d.get());
        CU(cudaMemcpyAsync(cls.data(), cls_d.get(), cls.size() * 4, cudaMemcpyDeviceToHost, b->stream.get()));
        CU(cudaStreamSynchronize(b->stream.get()));
        for (size_t k = 0; k < loc.size(); ++k) np->cls[wit[k]] = (uint8_t)std::min<u32>(cls[k], t.wit_class[wit[k]]);
    }
    build_pack_layout(t, np->L, np->cls.data());
    int rc;
    if ((rc = upload(np->pk_bit, np->L.bit_loc.data(), np->L.bit_loc.size() * 4))) return rc;
    if ((rc = upload(np->pk_u64, np->L.u64_loc.data(), np->L.u64_loc.size() * 4))) return rc;
    if ((rc = upload(np->pk_full, np->L.full_loc.data(), np->L.full_loc.size() * 4))) return rc;
    {
        std::lock_guard<std::mutex> lk(c->mu);
        c->narrow[b->device] = np;
    }
    out = np;
    return CW_OK;
}

// Packed transfer: entries the lowering proved to be one bit / <= 64 bits cross PCIe as that, the host expands
// them to the canonical 32-byte rows (zero-extension only - no field arithmetic happens on the CPU).  The batch
// moves in chunks through two staging buffers: while the worker threads expand chunk k, the pack kernel and the
// copy of chunk k + 1 run on the GPU / the copy engine.  CW_PACKED_D2H=0 forces the dense copy.
static int get_witness_packed_with(cw_batch *b, uint64_t *out, const PackLayout &L, const PackLayout &Lstatic,
                                   const NarrowPack *np, bool *flagged);
static int get_witness_packed(cw_batch *b, uint64_t *out, bool *done) {
    const Tape &t = b->c->tape;
    const PackLayout &Lstatic = b->c->pack_layout();
    *done = false;
    if (env_int("CW_PACKED_D2H", 1) == 0) return CW_OK;
    int rc;
    // Classes observed at run time (CW_PACK_OBSERVE=0: proven classes only).  Values that are bits or limbs without the
    // lowering being able to prove it - every xor of a hash circuit - then cross PCIe as bits / 8 bytes.  The first
    // transfer of a circuit looks at its batch; the pack kernel re-checks every value, a batch that shows a wider value
    // widens the layout and is sent again.
    std::shared_ptr<NarrowPack> np;
    if (env_int("CW_PACK_OBSERVE", 1) != 0 && (!Lstatic.u64_loc.empty() || !Lstatic.full_loc.empty())) {
        {
            std::lock_guard<std::mutex> lk(b->c->mu);
            auto it = b->c->narrow.find(b->device);
            if (it != b->c->narrow.end()) np = it->second;
        }
        if (!np && (rc = observe_classes(b, nullptr, np))) return rc;
    }
    for (int attempt = 0;; ++attempt) {
        const PackLayout &L = np ? np->L : Lstatic;
        if (L.words * 4 * 2 > (size_t)t.n_witness * 32) return CW_OK;   // not worth it: dense copy
        bool flagged = false;
        if ((rc = get_witness_packed_with(b, out, L, Lstatic, np.get(), &flagged))) return rc;
        if (!flagged) break;
        if (!np || attempt > 0) return CW_OK;   // a value exceeded its PROVEN class (never expected): dense copy
        std::shared_ptr<NarrowPack> wider;
        if ((rc = observe_classes(b, np, wider))) return rc;
        np = wider;
    }
    *done = true;
    return CW_OK;
}

// one pass of the packed transfer with layout L (staging buffers are sized for the proven layout, the widest)
static int get_witness_packed_with(cw_batch *b, uint64_t *out, const PackLayout &L, const PackLayout &Lstatic,
                                   const NarrowPack *np, bool *flagged) {
    const Tape &t = b->c->tape;
    int rc = ensure_pack_buffers(b, Lstatic);
    if (rc) return rc;
    CU(cudaMemsetAsync(b->pack_flag_d.get(), 0, 4, b->stream.get()));
    const size_t W = t.n_witness, cap = b->packed_cap;
    const size_t n_chunks = (b->batch + cap - 1) / cap;
    Pool &pool = Pool::get(device_numa_node(b->device));
    auto expand_chunk = [&](size_t k) {
        const size_t first = k * cap, cnt = std::min(cap, b->batch - first);
        const uint32_t *src = b->packed_h[k & 1].get();
        // item key = instance index: the rows of instance i of `out` are always written by the same (pinned) worker
        pool.parallel_for(cnt, first, [&](size_t i) { expand_record(L, src + i * L.words, out + (first + i) * W * 4); });
    };
    for (size_t k = 0; k < n_chunks; ++k) {
        const size_t first = k * cap, cnt = std::min(cap, b->batch - first);
        // staging buffer k & 1 was consumed by the expansion of chunk k - 2, which finished before chunk k - 1 was waited for
        if ((rc = pack_rows(b, L, (u32)first, (u32)cnt, b->packed_d[k & 1].get(), np))) return rc;
        CU(cudaMemcpyAsync(b->packed_h[k & 1].get(), b->packed_d[k & 1].get(), cnt * L.words * 4, cudaMemcpyDeviceToHost,
                           b->stream.get()));
        CU(cudaEventRecord(b->pack_ev[k & 1].get(), b->stream.get()));
        if (k > 0) {
            CU(cudaEventSynchronize(b->pack_ev[(k - 1) & 1].get()));
            expand_chunk(k - 1);
        }
    }
    int flag = 0;
    CU(cudaMemcpyAsync(&flag, b->pack_flag_d.get(), 4, cudaMemcpyDeviceToHost, b->stream.get()));
    CU(cudaStreamSynchronize(b->stream.get()));
    if (flag) {   // a value exceeded its class: the rows written so far are overwritten by the next attempt
        *flagged = true;
        return CW_OK;
    }
    expand_chunk(n_chunks - 1);
    b->last_d2h_bytes = (uint64_t)b->batch * L.words * 4;
    return CW_OK;
}

static int get_witness_impl(cw_batch *b, uint64_t *out) {
    const Tape &t = b->c->tape;
    CU(cudaSetDevice(b->device));
    bool done = false;
    int rc = get_witness_packed(b, out, &done);
    if (rc) return rc;
    if (done) return CW_OK;
    b->last_d2h_bytes = (uint64_t)b->batch * t.n_witness * 32;
    if (b->identity_layout()) {  // rows are read in place: pitched device-to-host copy
        CU(cudaMemcpy2DAsync(out, (size_t)t.n_witness * 32, b->slots.get(), (size_t)t.n_slots * 32, (size_t)t.n_witness * 32,
                             b->batch, cudaMemcpyDeviceToHost, b->stream.get()));
        CU(cudaStreamSynchronize(b->stream.get()));
        return CW_OK;
    }
    // dense rows, a bounded number of instances at a time
    const size_t row = (size_t)t.n_witness * 32;
    if (!b->dense_chunk_d) {
        size_t n = std::max<size_t>(1, std::min<size_t>(b->batch, ((size_t)512 << 20) / row));
        if ((rc = dev_alloc(b->dense_chunk_d, n * row))) return rc;
        b->dense_chunk_cap = n;
    }
    for (size_t first = 0; first < b->batch; first += b->dense_chunk_cap) {
        const size_t cnt = std::min(b->dense_chunk_cap, b->batch - first);
        if ((rc = expand_rows(b, (u32)first, (u32)cnt, b->dense_chunk_d.get()))) return rc;
        CU(cudaMemcpyAsync((uint8_t *)out + first * row, b->dense_chunk_d.get(), cnt * row, cudaMemcpyDeviceToHost,
                           b->stream.get()));
        CU(cudaStreamSynchronize(b->stream.get()));
    }
    return CW_OK;
}

int cw_batch_get_witness(cw_batch *b, uint64_t *out) {
    if (!b || !out) return fail(CW_EINVAL, "null argument");
    if (!b->ran) return fail(CW_ESTATE, "batch has not been run");
    if (b->async_active) return fail(CW_ESTATE, "a witness transfer of this batch is in flight (cw_batch_get_witness_wait)");
    return get_witness_impl(b, out);
}

// The same transfer on a helper thread: the caller may run OTHER batches (their own streams) meanwhile, so that the
// tape of batch k + 1 executes while the witnesses of batch k are packed, copied and expanded.
int cw_batch_get_witness_async(cw_batch *b, uint64_t *out) {
    if (!b || !out) return fail(CW_EINVAL, "null argument");
    if (!b->ran) return fail(CW_ESTATE, "batch has not been run");
    if (b->async_active) return fail(CW_ESTATE, "a witness transfer of this batch is already in flight");
    join_async(b);
    b->async_active = true;
    b->async_th = std::thread([b, out] {
        b->async_rc = get_witness_impl(b, out);
        b->async_err = g_err;  // (thread-local message of the helper thread)
    });
    return CW_OK;
}

int cw_batch_get_witness_wait(cw_batch *b) {
    if (!b) return fail(CW_EINVAL, "null argument");
    if (!b->async_active) return CW_OK;
    join_async(b);
    if (b->async_rc) return fail(b->async_rc, b->async_err);
    return CW_OK;
}

uint64_t cw_batch_last_d2h_bytes(const cw_batch *b) { return b ? b->last_d2h_bytes : 0; }

// The packed records themselves, for consumers that do not need 32-byte rows (layout: cw_circuit_pack_info)
int cw_batch_get_witness_packed(cw_batch *b, uint32_t *out_words) {
    if (!b || !out_words) return fail(CW_EINVAL, "null argument");
    if (!b->ran) return fail(CW_ESTATE, "batch has not been run");
    if (b->async_active) return fail(CW_ESTATE, "a witness transfer of this batch is in flight (cw_batch_get_witness_wait)");
    CU(cudaSetDevice(b->device));
    const PackLayout &L = b->c->pack_layout();
    int rc = ensure_pack_buffers(b, L);
    if (rc) return rc;
    CU(cudaMemsetAsync(b->pack_flag_d.get(), 0, 4, b->stream.get()));
    for (size_t first = 0; first < b->batch; first += b->packed_cap) {
        const size_t cnt = std::min(b->packed_cap, b->batch - first);
        if ((rc = pack_rows(b, L, (u32)first, (u32)cnt, b->packed_d[0].get()))) return rc;
        CU(cudaMemcpyAsync(out_words + first * L.words, b->packed_d[0].get(), cnt * L.words * 4, cudaMemcpyDeviceToHost,
                           b->stream.get()));
        CU(cudaStreamSynchronize(b->stream.get()));
    }
    int flag = 0;
    CU(cudaMemcpy(&flag, b->pack_flag_d.get(), 4, cudaMemcpyDeviceToHost));
    if (flag) return fail(CW_ESTATE, "a witness value exceeds the width the lowering proved for it");
    return CW_OK;
}

int cw_batch_witness_device(cw_batch *b, const uint64_t **dptr) {
    if (!b || !dptr) return fail(CW_EINVAL, "null argument");
    if (!b->ran) return fail(CW_ESTATE, "batch has not been run");
    CU(cudaSetDevice(b->device));
    int rc = dense_witness(b);
    if (rc) return rc;
    *dptr = (const uint64_t *)b->witness_d.get();
    return CW_OK;
}

int cw_batch_witness_strided(cw_batch *b, const uint64_t **dptr, uint64_t *stride_elems) {
    if (!b || !dptr || !stride_elems) return fail(CW_EINVAL, "null argument");
    if (!b->ran) return fail(CW_ESTATE, "batch has not been run");
    if (b->identity_layout()) {
        *dptr = (const uint64_t *)b->slots.get();
        *stride_elems = b->c->tape.n_slots;
        return CW_OK;
    }
    int rc = cw_batch_witness_device(b, dptr);
    *stride_elems = b->c->tape.n_witness;
    return rc;
}

void *cw_batch_stream(cw_batch *b) { return b ? (void *)b->stream.get() : nullptr; }

int cw_batch_last_ms(cw_batch *b, float *exec_ms, float *gather_ms) {
    if (!b || !b->ran) return fail(CW_ESTATE, "batch has not been run");
    CU(cudaSetDevice(b->device));
    CU(cudaEventSynchronize(b->ev[2].get()));
    if (exec_ms) CU(cudaEventElapsedTime(exec_ms, b->ev[0].get(), b->ev[1].get()));
    if (gather_ms) *gather_ms = 0.f;  // no gather pass: witness entries are written in place by the tape
    return CW_OK;
}

// the dense row of one instance, in host memory (for the .wtns writer and the log)
static int fetch_row(cw_batch *b, u32 inst, std::vector<uint64_t> &w) {
    const Tape &t = b->c->tape;
    CU(cudaSetDevice(b->device));
    w.resize((size_t)t.n_witness * 4);
    DevPtr<uint4> row;
    int rc;
    if ((rc = dev_alloc(row, (size_t)t.n_witness * 32))) return rc;
    if ((rc = expand_rows(b, inst, 1, row.get()))) return rc;
    CU(cudaMemcpyAsync(w.data(), row.get(), (size_t)t.n_witness * 32, cudaMemcpyDeviceToHost, b->stream.get()));
    CU(cudaStreamSynchronize(b->stream.get()));
    return CW_OK;
}

int cw_batch_wtns_bytes(cw_batch *b, uint32_t inst, uint8_t *out, size_t cap, size_t *len) {
    if (!b || inst >= b->batch) return fail(CW_EINVAL, "bad instance");
    if (!b->ran) return fail(CW_ESTATE, "batch has not been run");
    const Tape &t = b->c->tape;
    const size_t n8 = field_bytes(t.F);
    size_t need = 44 + n8 + n8 * (size_t)t.n_witness;
    if (len) *len = need;
    if (!out) return CW_OK;
    if (cap < need) return fail(CW_EINVAL, "buffer too small");
    std::vector<uint64_t> w;
    int rc = fetch_row(b, inst, w);
    if (rc) return rc;
    std::vector<uint8_t> bytes = wtns_bytes(t.F, w.data(), t.n_witness);
    memcpy(out, bytes.data(), need);
    return CW_OK;
}

int cw_batch_write_wtns(cw_batch *b, uint32_t inst, const char *path) {
    size_t need = 0;
    int rc = cw_batch_wtns_bytes(b, inst, nullptr, 0, &need);
    if (rc) return rc;
    std::vector<uint8_t> buf(need);
    if ((rc = cw_batch_wtns_bytes(b, inst, buf.data(), need, &need))) return rc;
    FILE *f = fopen(path, "wb");
    if (!f) return fail(CW_EIO, std::string("cannot open ") + path);
    size_t wr = fwrite(buf.data(), 1, need, f);
    fclose(f);
    return wr == need ? CW_OK : fail(CW_EIO, "short write");
}

// packed-record layout of the circuit: per witness entry (class << 30) | index - class 0: bit `index` of the plane
// section, 1: bit `index` of the extra-bit section, 2: u64 entry `index`, 3: full entry `index`; sections follow each
// other in that order; info = {words per instance, plane words, extra-bit words, u64 entries, full entries}
int cw_circuit_pack_info(const cw_circuit *c, uint64_t info[5], uint32_t *entry) {
    if (!c) return fail(CW_EINVAL, "null argument");
    const PackLayout &L = c->pack_layout();
    if (info) {
        info[0] = L.words;
        info[1] = L.n_plane_words;
        info[2] = L.n_bit_words;
        info[3] = L.u64_loc.size();
        info[4] = L.full_loc.size();
    }
    if (entry)
        for (const PackSeg &sg : L.segs)
            for (uint32_t j = 0; j < sg.count; ++j) entry[sg.start + j] = (sg.kind << 30) | (sg.src + j);
    return CW_OK;
}

// one packed record -> the n_witness canonical 32-byte rows of that instance (host memory; what cw_batch_get_witness
// does for every instance); `store_bits` 0 = widest vector stores of the CPU, or at most 128 / 256 / 512
int cw_circuit_expand_record(const cw_circuit *c, const uint32_t *record, uint64_t *rows, int store_bits) {
    if (!c || !record || !rows) return fail(CW_EINVAL, "null argument");
    expand_record(c->pack_layout(), record, rows, store_bits);
    return CW_OK;
}
const char *cw_host_expand_isa(void) { return expand_isa(); }
const char *cw_host_pool_info(void) { return Pool::get().describe(); }

// Host-side probe (no GPU): the expansion of `n_inst` packed records (all zero) into a freshly allocated row buffer on
// the worker pool, `reps` passes over the same buffer; mode 0 = expand_record, 1 = plain streaming fill of the same
// bytes (the memory system's ceiling for this access pattern), 2 = memset.  gbps[r] = bytes of rows written / time.
int cw_host_expand_bench(const cw_circuit *c, uint32_t n_inst, uint32_t reps, int mode, double *gbps) {
    if (!c || !gbps || !n_inst || !reps) return fail(CW_EINVAL, "bad argument");
    const PackLayout &L = c->pack_layout();
    const size_t W = c->tape.n_witness, row_bytes = W * 32;
    uint64_t *out = (uint64_t *)aligned_alloc(64, ((size_t)n_inst * row_bytes + 63) & ~(size_t)63);
    if (!out) return fail(CW_EINVAL, "out of host memory");
    std::vector<uint32_t> rec(L.words, 0);
    Pool &pool = Pool::get();
    for (uint32_t r = 0; r < reps; ++r) {
        auto t0 = std::chrono::steady_clock::now();
        pool.parallel_for(n_inst, 0, [&](size_t i) {
            uint64_t *dst = out + i * W * 4;
            if (mode == 0) expand_record(L, rec.data(), dst);
            else if (mode == 1) {
                const __m128i z = _mm_setzero_si128();
                for (size_t k = 0; k < W * 2; ++k) _mm_stream_si128((__m128i *)dst + k, z);
                _mm_sfence();
            } else memset(dst, 0, row_bytes);
        });
        double dt = std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
        gbps[r] = (double)n_inst * row_bytes / dt / 1e9;
    }
    free(out);
    return CW_OK;
}

// ---- R1CS -------------------------------------------------------------------------------------
int cw_r1cs_from_circuit(const cw_circuit *c, cw_r1cs **out) {
    if (!c || !out) return fail(CW_EINVAL, "null argument");
    cw_r1cs *r = new cw_r1cs();
    r->data = c->tape.r1cs;
    r->F = c->tape.F;
    *out = r;
    return CW_OK;
}
int cw_r1cs_load(const char *path, cw_r1cs **out) {
    if (!path || !out) return fail(CW_EINVAL, "null argument");
    auto r = std::make_unique<cw_r1cs>();
    try {
        read_r1cs(path, r->data);
    } catch (const std::exception &e) {
        return fail(CW_EFORMAT, e.what());
    }
    r->F = make_field(r->data.prime_id);
    *out = r.release();
    return CW_OK;
}
int cw_r1cs_write(const cw_r1cs *r, const char *path, uint32_t n_pub_out, uint32_t n_pub_in, uint32_t n_prv_in) {
    if (!r || !path) return fail(CW_EINVAL, "null argument");
    try {
        R1csData d = r->data;  // CW_KEEP: the count the circuit / the loaded file carries
        if (n_pub_out != CW_KEEP) d.n_pub_out = n_pub_out;
        if (n_pub_in != CW_KEEP) d.n_pub_in = n_pub_in;
        if (n_prv_in != CW_KEEP) d.n_prv_in = n_prv_in;
        write_r1cs(d, r->F, path);
    } catch (const std::exception &e) {
        return fail(CW_EIO, e.what());
    }
    return CW_OK;
}
int cw_r1cs_info(const cw_r1cs *r, uint64_t *n_wires, uint64_t *n_constraints, uint64_t *nnz, int *prime_id) {
    if (!r) return fail(CW_EINVAL, "null argument");
    if (n_wires) *n_wires = r->data.n_wires;
    if (n_constraints) *n_constraints = r->data.n_constraints;
    if (nnz) *nnz = r->data.col.size();
    if (prime_id) *prime_id = r->data.prime_id;
    return CW_OK;
}
void cw_r1cs_destroy(cw_r1cs *r) {
    if (!r) return;
    cw_r1cs_destroy(r->eval_twin.release());
    cw_r1cs_destroy(r->qap_twin.release());
    for (auto it = r->dev.begin(); it != r->dev.end(); it = r->dev.erase(it)) cudaSetDevice(it->first.device);
    delete r;
}

// The CSR compiled for one value layout (r1cs_compile.cpp), uploaded.
static int compile_r1cs(cw_r1cs *r, const cw_circuit *layout, DevR1cs &d) {
    R1csCompiled h;
    try {
        compile_r1cs_host(r->data, r->F, layout ? &layout->tape : nullptr, r->no_bool_rows,
                          !r->no_bool_rows && env_int("CW_R1CS_SMALL", 1) != 0, h);
    } catch (const std::exception &e) {
        return fail(CW_EINVAL, e.what());
    }
    int rc;
    static_assert(sizeof(R1csTerm) == sizeof(uint4), "term records are read as uint4");
    d.n_general = (u32)h.perm.size();
    d.n_small = (u32)h.perm_small.size();
    d.n_bool = (u32)h.bool_loc.size();
    d.n_terms = h.n_terms;
    d.mean_row_terms = h.mean_row_terms;
    if ((rc = upload(d.terms, h.terms.data(), h.terms.size() * sizeof(uint4)))) return rc;
    if ((rc = upload(d.bool_loc, h.bool_loc.data(), h.bool_loc.size() * 4))) return rc;
    if ((rc = upload(d.bool_row, h.bool_row.data(), h.bool_row.size() * 4))) return rc;
    if ((rc = upload(d.row_ptr, h.row_ptr.data(), h.row_ptr.size() * 8))) return rc;
    if ((rc = upload(d.dictM, h.dictM.data(), h.dictM.size() * 32))) return rc;
    if ((rc = upload(d.perm, h.perm.data(), h.perm.size() * 4))) return rc;
    if ((rc = upload(d.perm_small, h.perm_small.data(), h.perm_small.size() * 4))) return rc;
    static_assert(sizeof(R1csSmallRec) == sizeof(uint2), "integer-row records are read as uint2");
    if ((rc = upload(d.sgroups, h.sgroups.data(), h.sgroups.size() * 4))) return rc;
    if ((rc = upload(d.srecs, h.srecs.data(), h.srecs.size() * sizeof(uint2)))) return rc;
    if ((rc = upload(d.sbrow, h.sbrow.data(), h.sbrow.size() * 4))) return rc;
    d.general = {d.row_ptr.get(), d.terms.get(), d.dictM.get(), d.perm.get(), d.n_general, (u32)r->data.prime_id};
    d.integer = d.general;
    d.integer.perm = d.perm_small.get();
    d.integer.n_rows = d.n_small;
    d.integer_recs = {d.sgroups.get(), d.srecs.get(), d.sbrow.get()};
    return CW_OK;
}

// the CSR of r for the value layout of `layout` (nullptr: dense rows) on `device`, compiled on first use
static int get_dev_r1cs(cw_r1cs *r, int device, const cw_circuit *layout, const DevR1cs *&out) {
    std::lock_guard<std::mutex> lk(r->mu);
    R1csKey key{device, layout ? layout->serial : 0};
    auto it = r->dev.find(key);
    if (it == r->dev.end()) {
        DevR1cs d;
        int rc = compile_r1cs(r, layout, d);
        if (rc) return rc;
        it = r->dev.emplace(key, std::move(d)).first;
    }
    out = &it->second;
    return CW_OK;
}

// launches on `stream`; fb_d[batch] must hold ~0 on entry; `wide` = (n_small + 31) / 32 + 1 words of scratch for the rows the
// integer-row kernel hands to the general one
static int launch_r1cs(cw_r1cs *r, const DevR1cs &d, const StoreDev &S, cudaStream_t stream, unsigned long long *fb_d,
                       const EvalOut *eval, u32 *wide) {
    const int prime_id = r->data.prime_id;
    const u32 bt_mask = (1u << S.bt_log2) - 1u;
    const u32 n_tiles = eval ? ((eval->first + eval->count + bt_mask) >> S.bt_log2) - (eval->first >> S.bt_log2)
                             : (S.batch + bt_mask) >> S.bt_log2;
    auto grid = [&](u32 rows) { return grid_for((uint64_t)rows << S.bt_log2, 256, 8, n_tiles); };
    if (d.n_general) {
        const dim3 g = grid(d.n_general);
        // long rows: many resident warps (48 registers); short rows: the unspilled build
        const bool lean = env_int("CW_R1CS_LEAN", d.mean_row_terms >= 12 ? 1 : 0) != 0;
        const EvalOut eo = eval ? *eval : EvalOut();
        with_prime(prime_id, [&](auto pr) {
            constexpr int PR = decltype(pr)::value;
            if (eval) {
                r1cs_check_kernel<PR, 3, true, false><<<g, 256, 0, stream>>>(d.general, S, fb_d, eo, nullptr);
                return;
            }
            if constexpr (PR >= 0)   // (the lean build exists for bn128 and bls12381)
                if (lean) {
                    r1cs_check_kernel<PR, 5, false, false><<<g, 256, 0, stream>>>(d.general, S, fb_d, eo, nullptr);
                    return;
                }
            r1cs_check_kernel<PR, 3, false, false><<<g, 256, 0, stream>>>(d.general, S, fb_d, eo, nullptr);
        });
    }
    if (d.n_small) {
        // rows that are small by shape: over the integers first; the rows in which a value turned out wide (bitmap) go
        // through the general kernel afterwards
        if (!wide || eval) return fail(CW_ESTATE, "integer rows need their scratch bitmap");
        CU(cudaMemsetAsync(wide, 0, (((size_t)d.n_small + 31) / 32 + 1) * 4, stream));
        const dim3 g = grid(d.n_small);
        if (S.bt_log2 == 0) r1cs_small_kernel<true><<<g, 256, 0, stream>>>(d.integer, d.integer_recs, S, fb_d, wide);
        else r1cs_small_kernel<false><<<g, 256, 0, stream>>>(d.integer, d.integer_recs, S, fb_d, wide);
        with_prime(prime_id, [&](auto pr) {
            r1cs_check_kernel<decltype(pr)::value, 3, false, true><<<g, 256, 0, stream>>>(d.integer, S, fb_d, EvalOut(), wide);
        });
    }
    if (d.n_bool && !eval)
        r1cs_bool_kernel<<<grid(d.n_bool), 256, 0, stream>>>(d.bool_loc.get(), d.bool_row.get(), d.n_bool, S, fb_d);
    CU(cudaGetLastError());
    return CW_OK;
}

int cw_r1cs_check(cw_r1cs *r, const uint64_t *witness, int is_device_ptr, uint32_t batch, int device,
                  int64_t *first_bad, float *kernel_ms) {
    if (!r) return fail(CW_EINVAL, "bad argument");
    return cw_r1cs_check_strided(r, witness, r->data.n_wires, is_device_ptr, batch, device, first_bad, kernel_ms);
}

// the check of store S on `stream` (launch_r1cs), timed by events around the kernels; first_bad[i] = the first violated
// row of instance i, or -1
static int check_store(cw_r1cs *r, const DevR1cs &d, const StoreDev &S, cudaStream_t stream, unsigned long long *fb_d,
                       u32 *wide, int64_t *first_bad, float *kernel_ms) {
    Event e0, e1;
    int rc;
    if ((rc = make_event(e0)) || (rc = make_event(e1))) return rc;
    CU(cudaMemsetAsync(fb_d, 0xFF, (size_t)S.batch * 8, stream));
    CU(cudaEventRecord(e0.get(), stream));
    if ((rc = launch_r1cs(r, d, S, stream, fb_d, nullptr, wide))) return rc;
    CU(cudaEventRecord(e1.get(), stream));
    std::vector<unsigned long long> fb(S.batch);
    CU(cudaMemcpyAsync(fb.data(), fb_d, (size_t)S.batch * 8, cudaMemcpyDeviceToHost, stream));
    CU(cudaStreamSynchronize(stream));
    float ms = 0;
    CU(cudaEventElapsedTime(&ms, e0.get(), e1.get()));
    if (kernel_ms) *kernel_ms = ms;
    for (u32 i = 0; i < S.batch; ++i) first_bad[i] = fb[i] == ~0ull ? -1 : (int64_t)fb[i];
    return CW_OK;
}

// dense witness rows handed in by the caller (host or device memory)
int cw_r1cs_check_strided(cw_r1cs *r, const uint64_t *witness, uint64_t stride_elems, int is_device_ptr, uint32_t batch,
                          int device, int64_t *first_bad, float *kernel_ms) {
    if (!r || !witness || !first_bad || batch == 0 || stride_elems < r->data.n_wires || stride_elems >> 32)
        return fail(CW_EINVAL, "bad argument");
    if (is_device_ptr && ((uintptr_t)witness & 31u))
        return fail(CW_EINVAL, "device witness pointer must be 32-byte aligned (elements are read with 256-bit loads)");
    int rc = ensure_device(device);
    if (rc) return rc;
    const DevR1cs *d;
    if ((rc = get_dev_r1cs(r, device, nullptr, d))) return rc;
    const R1csData &R = r->data;
    const void *w_d = witness;
    DevPtr<uint4> tmp;
    if (!is_device_ptr) {
        if ((rc = dev_alloc(tmp, (size_t)batch * R.n_wires * 32))) return rc;
        CU(cudaMemcpy2D(tmp.get(), (size_t)R.n_wires * 32, witness, (size_t)stride_elems * 32, (size_t)R.n_wires * 32, batch,
                        cudaMemcpyHostToDevice));
        w_d = tmp.get();
        stride_elems = R.n_wires;
    }
    DevPtr<unsigned long long> fb_d;
    DevPtr<u32> wide_d;
    if ((rc = dev_alloc(fb_d, (size_t)batch * 8))) return rc;
    if (d->n_small && (rc = dev_alloc(wide_d, (((size_t)d->n_small + 31) / 32 + 1) * 4))) return rc;
    return check_store(r, *d, dense_store(w_d, stride_elems, batch), nullptr, fb_d.get(), wide_d.get(), first_bad, kernel_ms);
}

// The witnesses of a batch where the tape left them (resident slots + bit plane, any tile layout): no dense rows
// are materialised, plane bits are read as bits, recomposition sums as words.  Runs on the batch's stream, behind
// the tape; the per-instance result buffer belongs to the batch (no allocation per call).
int cw_r1cs_check_batch(cw_r1cs *r, cw_batch *b, int64_t *first_bad, float *kernel_ms) {
    if (!r || !b || !first_bad) return fail(CW_EINVAL, "null argument");
    if (!b->ran) return fail(CW_ESTATE, "batch has not been run");
    if (r->data.prime_id != b->c->tape.F.prime_id) return fail(CW_EINVAL, "the R1CS and the batch use different primes");
    CU(cudaSetDevice(b->device));
    const DevR1cs *d;
    int rc = get_dev_r1cs(r, b->device, b->c, d);
    if (rc) return rc;
    if (d->n_small > b->r1cs_wide_rows) {   // scratch of the integer rows: grows with the largest R1CS this batch has checked
        CU(cudaStreamSynchronize(b->stream.get()));
        b->r1cs_wide_d.reset();
        b->r1cs_wide_rows = 0;
        if ((rc = dev_alloc(b->r1cs_wide_d, (((size_t)d->n_small + 31) / 32 + 1) * 4))) return rc;
        b->r1cs_wide_rows = d->n_small;
    }
    return check_store(r, *d, b->store(), b->stream.get(), b->fb_d.get(), b->r1cs_wide_d.get(), first_bad, kernel_ms);
}

static int copy_text(const std::string &msg, char *buf, size_t cap, size_t *len) {
    if (len) *len = msg.size();
    if (buf && cap) {
        const size_t n = std::min(msg.size(), cap - 1);
        memcpy(buf, msg.data(), n);
        buf[n] = 0;
    }
    return CW_OK;
}

int cw_circuit_format_log(const cw_circuit *c, const uint64_t *witness, char *buf, size_t cap, size_t *len) {
    if (!c || !witness) return fail(CW_EINVAL, "null argument");
    return copy_text(format_log(c->tape, witness), buf, cap, len);
}

int cw_batch_log(cw_batch *b, uint32_t inst, char *buf, size_t cap, size_t *len) {
    if (!b || inst >= b->batch) return fail(CW_EINVAL, "bad instance");
    if (!b->ran) return fail(CW_ESTATE, "batch has not been run");
    const Tape &t = b->c->tape;
    if (t.log_args.empty()) return copy_text(std::string(), buf, cap, len);
    std::vector<uint64_t> w;
    int rc = fetch_row(b, inst, w);
    if (rc) return rc;
    return copy_text(format_log(t, w.data()), buf, cap, len);
}

int cw_circuit_assert_info(const cw_circuit *c, uint32_t assert_no, char *buf, size_t cap, size_t *len) {
    if (!c) return fail(CW_EINVAL, "null argument");
    const Tape &t = c->tape;
    if (assert_no >= t.assert_tid.size()) return fail(CW_EINVAL, "no such assert (or a circuit without its description: broadcast)");
    std::string msg = "Failed assert in template/function " + t.tmpl_names[t.assert_tid[assert_no]];
    if (!t.sym.empty()) {
        // the component whose signals start at assert_start: walk down from main by signal ranges (own signals first, then
        // the sub-components in creation order - the numbering of the whole description)
        std::string trace = "main";
        uint32_t tid = t.sym_main;
        uint64_t start = 1;   // (signal 0 is the constant one)
        const uint64_t want = t.assert_start[assert_no];
        while (start != want) {
            const Tape::SymTemplate &st = t.sym[tid];
            uint64_t off = start + st.n_own;
            bool down = false;
            for (size_t i = 0; i < st.subs.size(); ++i) {
                const uint64_t n = t.sym[st.subs[i]].total_signals;
                if (want >= off && want < off + n) {
                    trace += "." + st.sub[i];
                    tid = st.subs[i];
                    start = off;
                    down = true;
                    break;
                }
                off += n;
            }
            if (!down) return fail(CW_EINVAL, "assert site outside the component tree");
        }
        msg += ". Followed trace of components: " + trace;
    }
    return copy_text(msg, buf, cap, len);
}

int cw_r1cs_compiled_info(cw_r1cs *r, cw_batch *b, int device, uint64_t info[4]) {
    if (!r || !info) return fail(CW_EINVAL, "null argument");
    int rc = b ? CW_OK : ensure_device(device);
    if (rc) return rc;
    if (b) CU(cudaSetDevice(b->device));
    const DevR1cs *d;
    if ((rc = get_dev_r1cs(r, b ? b->device : device, b ? b->c : nullptr, d))) return rc;
    info[0] = d->n_general;
    info[1] = d->n_small;
    info[2] = d->n_bool;
    info[3] = d->n_terms;
    return CW_OK;
}

// r's constraints compiled with every row general (no boolean-row special cases): the twin of cw_r1cs_eval_batch, or
// with `qap` that of the quotient, which appends the rows a_{m+j} = 1 * w_j (j <= n_public)
static cw_r1cs *general_twin(cw_r1cs *r, bool qap, u32 n_public = 0) {
    std::lock_guard<std::mutex> lk(r->mu);
    std::unique_ptr<cw_r1cs> &twin = qap ? r->qap_twin : r->eval_twin;
    if (twin) return twin.get();
    auto t = std::make_unique<cw_r1cs>();
    t->data = r->data;
    t->F = r->F;
    t->no_bool_rows = true;
    if (qap) {
        R1csData &D = t->data;
        D.has_custom_gates = false;
        D.gates_used.clear();
        D.gates_applied.clear();
        const U256 one = u256_from_u64(1);
        u32 one_idx = (u32)D.dict.size();
        for (size_t i = 0; i < D.dict.size(); ++i)
            if (D.dict[i] == one) { one_idx = (u32)i; break; }
        if (one_idx == D.dict.size()) D.dict.push_back(one);
        for (u32 j = 0; j <= n_public; ++j) {   // row_ptr[3 m] (the end of the last row) is the start of the new row's A block
            D.col.push_back(j);
            D.coef.push_back(one_idx);
            for (int k = 0; k < 3; ++k) D.row_ptr.push_back(D.col.size());
        }
        D.n_constraints += n_public + 1;
    }
    twin = std::move(t);
    return twin.get();
}

// A.w, B.w, C.w of every constraint for instances [first, first + count) of a batch, left in device memory for a
// prover (the QAP evaluation / rapidsnark-style pipeline that follows witness generation): three arrays
// [count][n_constraints][4 x u64], canonical.  Rows the check treats specially (boolean rows) are evaluated like
// all others here.
int cw_r1cs_eval_batch(cw_r1cs *r, cw_batch *b, uint32_t first, uint32_t count, uint64_t *a_dev, uint64_t *b_dev,
                       uint64_t *c_dev) {
    if (!r || !b || !a_dev || !b_dev || !c_dev || (uint64_t)first + count > b->batch || count == 0)
        return fail(CW_EINVAL, "bad argument");
    if (((uintptr_t)a_dev | (uintptr_t)b_dev | (uintptr_t)c_dev) & 31u) return fail(CW_EINVAL, "outputs must be 32-byte aligned");
    if (!b->ran) return fail(CW_ESTATE, "batch has not been run");
    if (r->data.prime_id != b->c->tape.F.prime_id) return fail(CW_EINVAL, "the R1CS and the batch use different primes");
    CU(cudaSetDevice(b->device));
    cw_r1cs *all = general_twin(r, false);
    const DevR1cs *d;
    int rc = get_dev_r1cs(all, b->device, b->c, d);
    if (rc) return rc;
    EvalOut eo;
    eo.a = (uint4 *)a_dev;
    eo.b = (uint4 *)b_dev;
    eo.c = (uint4 *)c_dev;
    eo.stride = r->data.n_constraints;
    eo.first = first;
    eo.count = count;
    CU(cudaMemsetAsync(b->fb_d.get(), 0xFF, (size_t)b->batch * 8, b->stream.get()));
    return launch_r1cs(all, *d, b->store(), b->stream.get(), b->fb_d.get(), &eo, nullptr);
}

// ---- Groth16 quotient evaluations (the QAP step every Groth16 prover starts with) --------------------------------
// Domain n = 2^k >= m + nPublic + 1 with k + 1 <= s (the 2-adicity of q - 1).  Values on the domain: a_i = (A.w)_i and
// b_i = (B.w)_i for i < m, a_{m+j} = w_j for j <= nPublic, zero elsewhere; c = a o b.  Each goes to the odd coset
// (inverse NTT, times w_2n^i, NTT) and h = a' b' - c'.
static int qap_domain(const cw_r1cs *r, u32 &log_n, u32 &n_public) {
    const R1csData &R = r->data;
    const uint64_t np = (uint64_t)R.n_pub_out + R.n_pub_in;
    if (R.n_constraints == 0) return fail(CW_EINVAL, "the R1CS has no constraints");
    if (np + 1 > R.n_wires) return fail(CW_EINVAL, "more public signals than wires");
    const uint64_t rows = R.n_constraints + np + 1;
    u32 k = 0;
    while ((1ull << k) < rows) ++k;
    const u32 s = ntt_two_adicity(r->F);
    if (k + 1 > s) return fail(CW_EINVAL, "the prime's 2-adicity (" + std::to_string(s) + ") admits no domain of 2^" +
                                              std::to_string(k) + " points with its odd coset");
    log_n = k;
    n_public = (u32)np;
    return CW_OK;
}

// twiddle and coset-scale tables of one (device, prime, log_n), Montgomery images (ntt.cuh: ntt_tables)
struct NttTables {
    DevPtr<u32> tw, shi, slo;
};
static std::mutex g_ntt_mu;
// (device, prime, log_n): kept for the process, and never destroyed (no device calls at exit)
static auto &g_ntt_tables = *new std::map<std::tuple<int, int, u32>, NttTables>();

static int ntt_tables_for(int device, int prime_id, u32 log_n, const NttTables *&out) {
    std::lock_guard<std::mutex> lk(g_ntt_mu);
    auto key = std::make_tuple(device, prime_id, log_n);
    auto it = g_ntt_tables.find(key);
    if (it == g_ntt_tables.end()) {
        std::vector<U256> tw, shi, slo;
        ntt_tables(make_field(prime_id), log_n, tw, shi, slo);
        NttTables t;
        int rc;
        if ((rc = upload(t.tw, tw.data(), tw.size() * 32))) return rc;
        if ((rc = upload(t.shi, shi.data(), shi.size() * 32))) return rc;
        if ((rc = upload(t.slo, slo.data(), slo.size() * 32))) return rc;
        it = g_ntt_tables.emplace(key, std::move(t)).first;
    }
    out = &it->second;
    return CW_OK;
}

static int launch_ntt_passes(const NttPass *ps, u32 np, bool dit, const NttVecs &V, const NttTables &tb, int prime_id,
                             cudaStream_t stream) {
    using Kernel = void (*)(NttPass, NttVecs, const u32 *, const u32 *, const u32 *, u32);
    const Kernel kern = with_prime(prime_id, [&](auto pr) -> Kernel {
        return dit ? ntt_pass_kernel<decltype(pr)::value, true> : ntt_pass_kernel<decltype(pr)::value, false>;
    });
    const u32 prime = (u32)prime_id;
    CU(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, 32 << NTT_TILE_LOG));
    for (u32 k = 0; k < np; ++k) {
        const NttPass &p = ps[k];
        const u32 tiles = 1u << (p.log_n - p.b - p.log_g);
        dim3 grid(tiles, std::min<u32>(V.n_vec, 65535u));
        kern<<<grid, NTT_THREADS, (size_t)32 << (p.b + p.log_g), stream>>>(p, V, tb.tw.get(), tb.shi.get(), tb.slo.get(), prime);
    }
    return CW_OK;
}

// the vectors of V (d0 + v n for v < n0, then d1) through one transform of mode NTT_MODE_*, on `stream`
static int run_ntt(int device, int prime_id, u32 log_n, const NttVecs &V, int mode, cudaStream_t stream) {
    const NttTables *tb;
    int rc = ntt_tables_for(device, prime_id, log_n, tb);
    if (rc) return rc;
    NttPass dif[NTT_MAX_PASSES], dit[NTT_MAX_PASSES];
    const u32 lg_lo = ntt_lg_lo(log_n);
    const u32 scale = mode == NTT_MODE_FORWARD ? NTT_SCALE_NONE : mode == NTT_MODE_INVERSE ? NTT_SCALE_CONST : NTT_SCALE_COSET;
    const u32 nd = ntt_plan(log_n, false, mode != NTT_MODE_FORWARD, scale, lg_lo, dif);
    const u32 nt = mode == NTT_MODE_COSET ? ntt_plan(log_n, true, 0u, NTT_SCALE_NONE, lg_lo, dit) : 0u;
    if ((rc = launch_ntt_passes(dif, nd, false, V, *tb, prime_id, stream))) return rc;
    if (mode == NTT_MODE_COSET) {
        if ((rc = launch_ntt_passes(dit, nt, true, V, *tb, prime_id, stream))) return rc;
    } else {
        ntt_bitrev_kernel<<<grid_for(1ull << log_n, 256, 8, V.n_vec), 256, 0, stream>>>(V, log_n);
    }
    CU(cudaGetLastError());
    return CW_OK;
}

int cw_r1cs_qap_info(const cw_r1cs *r, uint32_t *log2_n, uint32_t *n_public) {
    if (!r) return fail(CW_EINVAL, "null argument");
    u32 k = 0, np = 0;
    int rc = qap_domain(r, k, np);
    if (rc) return rc;
    if (log2_n) *log2_n = k;
    if (n_public) *n_public = np;
    return CW_OK;
}

// the domain values of the window [first, first + count) of store S, transformed and joined into h (on `stream`)
static int quotient_on_store(cw_r1cs *r, int device, const cw_circuit *layout, const StoreDev &S, u32 first, u32 count,
                             uint64_t *h_dev, uint64_t *scratch_dev, unsigned long long *fb_d, cudaStream_t stream) {
    u32 k = 0, np = 0;
    int rc = qap_domain(r, k, np);
    if (rc) return rc;
    cw_r1cs *t = general_twin(r, true, np);
    const DevR1cs *d;
    if ((rc = get_dev_r1cs(t, device, layout, d))) return rc;
    const uint64_t n = 1ull << k, rows = t->data.n_constraints;
    uint4 *A = (uint4 *)h_dev, *B = (uint4 *)scratch_dev, *Cc = B + 2 * (size_t)count * n;
    if (rows < n)
        for (uint4 *p : {A, B, Cc}) CU(cudaMemset2DAsync(p + 2 * rows, n * 32, 0, (n - rows) * 32, count, stream));
    EvalOut eo;
    eo.a = A;
    eo.b = B;
    eo.c = Cc;
    eo.stride = n;
    eo.first = first;
    eo.count = count;
    eo.ab = 1u;
    if ((rc = launch_r1cs(t, *d, S, stream, fb_d, &eo, nullptr))) return rc;
    NttVecs V;
    V.d0 = A;
    V.d1 = B;
    V.n0 = count;
    V.n_vec = 3 * count;
    if ((rc = run_ntt(device, r->data.prime_id, k, V, NTT_MODE_COSET, stream))) return rc;
    const size_t tot = (size_t)count * n;
    const u32 prime = (u32)r->data.prime_id;
    with_prime(r->data.prime_id, [&](auto pr) {
        qap_join_kernel<decltype(pr)::value><<<grid_for(tot, 256, 8), 256, 0, stream>>>(A, A, B, Cc, tot, prime);
    });
    CU(cudaGetLastError());
    return CW_OK;
}

int cw_r1cs_quotient_batch(cw_r1cs *r, cw_batch *b, uint32_t first, uint32_t count, uint64_t *h_dev, uint64_t *scratch_dev) {
    if (!r || !b || !h_dev || !scratch_dev || count == 0 || (uint64_t)first + count > b->batch)
        return fail(CW_EINVAL, "bad argument");
    if (((uintptr_t)h_dev | (uintptr_t)scratch_dev) & 31u) return fail(CW_EINVAL, "h and scratch must be 32-byte aligned");
    if (!b->ran) return fail(CW_ESTATE, "batch has not been run");
    if (r->data.prime_id != b->c->tape.F.prime_id) return fail(CW_EINVAL, "the R1CS and the batch use different primes");
    CU(cudaSetDevice(b->device));
    CU(cudaMemsetAsync(b->fb_d.get(), 0xFF, (size_t)b->batch * 8, b->stream.get()));
    return quotient_on_store(r, b->device, b->c, b->store(), first, count, h_dev, scratch_dev, b->fb_d.get(), b->stream.get());
}

int cw_r1cs_quotient_strided(cw_r1cs *r, const uint64_t *witness_dev, uint64_t stride_elems, uint32_t count, int device,
                             uint64_t *h_dev, uint64_t *scratch_dev) {
    if (!r || !witness_dev || !h_dev || !scratch_dev || count == 0 || stride_elems < r->data.n_wires || stride_elems >> 32)
        return fail(CW_EINVAL, "bad argument");
    if (((uintptr_t)witness_dev | (uintptr_t)h_dev | (uintptr_t)scratch_dev) & 31u)
        return fail(CW_EINVAL, "device pointers must be 32-byte aligned");
    int rc = ensure_device(device);
    if (rc) return rc;
    DevPtr<unsigned long long> fb_d;
    if ((rc = dev_alloc(fb_d, (size_t)count * 8))) return rc;
    if ((rc = quotient_on_store(r, device, nullptr, dense_store(witness_dev, stride_elems, count), 0, count, h_dev, scratch_dev,
                                fb_d.get(), 0)))
        return rc;
    CU(cudaStreamSynchronize(0));
    return CW_OK;
}

int cw_fr_ntt_batch(int prime_id, uint32_t log2_n, uint32_t count, uint64_t *data_dev, int mode, int device) {
    if (prime_id < 0 || prime_id >= CW_N_PRIMES || !data_dev || count == 0 || mode < CW_NTT_FORWARD || mode > CW_NTT_COSET)
        return fail(CW_EINVAL, "bad argument");
    if ((uintptr_t)data_dev & 31u) return fail(CW_EINVAL, "data must be 32-byte aligned");
    const u32 s = ntt_two_adicity(make_field(prime_id));
    if (log2_n < 1 || log2_n > 27 || log2_n + 1 > s)
        return fail(CW_EINVAL, "log2_n must lie in [1, min(27, s - 1)]; the prime's 2-adicity s is " + std::to_string(s));
    int rc = ensure_device(device);
    if (rc) return rc;
    NttVecs V;
    V.d0 = (uint4 *)data_dev;
    V.d1 = nullptr;
    V.n0 = count;
    V.n_vec = count;
    static_assert(CW_NTT_FORWARD == NTT_MODE_FORWARD && CW_NTT_INVERSE == NTT_MODE_INVERSE && CW_NTT_COSET == NTT_MODE_COSET,
                  "transform modes");
    if ((rc = run_ntt(device, prime_id, log2_n, V, mode, 0))) return rc;
    CU(cudaStreamSynchronize(0));
    return CW_OK;
}

// ---- multi-scalar multiplication on G1 of BN254 (msm.cuh) -------------------------------------------------------------
struct cw_g1_bases {
    int device = 0;
    uint64_t n = 0;
    DevPtr<u32> pts;   // [n][16] u32: Montgomery x, y; (0, 0) = infinity
};

static const uint64_t MSM_MAX_N = 1ull << 26;
static const size_t MSM_CHUNK_BYTES = (size_t)2 << 30;   // scratch of one chunk of instances, about

// the scratch of one chunk of `chunk` instances: offsets into the caller's buffer (each 256-byte aligned)
struct MsmPlan {
    u32 c = 0, W = 0, B = 0, chunk = 0;
    uint64_t n = 0, items = 0, slots[2] = {0, 0};
    size_t keys[2], vals[2], cub, cub_bytes = 0, buckets, lv_keys[2], lv_pts[2], segs, wins, total = 0;
};
static u32 msm_seg_bits(u32 segs) {   // bits of the largest segment index
    u32 b = 0;
    while (b < 32 && ((uint64_t)1 << b) < segs) ++b;
    return b;
}
// pt_bytes: the bucket type's size, sizeof(Xyzz) for G1 and MSM_G2_POINT_BYTES for G2
static int msm_plan(uint64_t n, u32 chunk, MsmPlan &p, size_t pt_bytes) {
    p.n = n;
    const int cw = env_int("CW_MSM_WINDOW", 0);   // (window sweeps: scripts/msm_bench.py)
    p.c = cw >= (int)MSM_MIN_C && cw <= (int)MSM_MAX_C ? (u32)cw : msm_window_bits(n);
    p.W = msm_windows(p.c);
    p.B = 1u << (p.c - 1);
    p.chunk = chunk;
    p.items = (uint64_t)chunk * p.W * n;
    p.slots[0] = msm_level_out(p.items);
    p.slots[1] = msm_level_out(p.slots[0]);
    CU(cub::DeviceRadixSort::SortPairs(nullptr, p.cub_bytes, (const u32 *)nullptr, (u32 *)nullptr, (const u32 *)nullptr,
                                       (u32 *)nullptr, (int)p.items, 0, (int)(p.c + msm_seg_bits(chunk * p.W))));
    size_t at = 0;
    auto take = [&](size_t bytes) {
        const size_t o = at;
        at += (bytes + 255) & ~(size_t)255;
        return o;
    };
    for (int k = 0; k < 2; ++k) {
        p.keys[k] = take(p.items * 4);
        p.vals[k] = take(p.items * 4);
    }
    p.cub = take(p.cub_bytes);
    p.buckets = take((size_t)chunk * p.W * p.B * pt_bytes);
    for (int k = 0; k < 2; ++k) {
        p.lv_keys[k] = take(p.slots[k] * 4);
        p.lv_pts[k] = take(p.slots[k] * pt_bytes);
    }
    const u32 m = p.B < MSM_SEG ? p.B : MSM_SEG;
    p.segs = take((size_t)chunk * p.W * (p.B / m) * pt_bytes);
    p.wins = take((size_t)chunk * p.W * pt_bytes);
    p.total = at;
    return CW_OK;
}
// the chunk size for `count` instances of n points: bounded by MSM_CHUNK_BYTES, the 32-bit keys and int item counts
static int msm_plan_for(uint64_t n, u32 count, MsmPlan &p, size_t pt_bytes = sizeof(Xyzz)) {
    MsmPlan one;
    int rc = msm_plan(n, 1, one, pt_bytes);
    if (rc) return rc;
    uint64_t chunk = std::max<uint64_t>(1, MSM_CHUNK_BYTES / one.total);
    chunk = std::min<uint64_t>(chunk, count);
    chunk = std::min<uint64_t>(chunk, ((1ull << (32 - one.c)) - 1) / one.W);
    chunk = std::min<uint64_t>(chunk, std::max<uint64_t>(1, (uint64_t)INT32_MAX / (one.W * n)));
    return msm_plan(n, (u32)chunk, p, pt_bytes);
}

// n affine G1 points [n][2][4] u64 - canonical, or Montgomery images when `mont` (as a .zkey stores them) - checked on
// the host: (0, 0) is infinity, anything else has both coordinates below q and lies on the curve; out receives the
// Montgomery images the MSM reads.  `what` prefixes the messages, which name the first bad index.
static int g1_points_mont(const uint64_t *points, uint64_t n, bool mont, const std::string &what, std::vector<U256> &out) {
    const FieldParams F = make_field(MSM_PRIME);
    const U256 three = F.to_mont(u256_from_u64(3));
    out.assign(2 * n, U256());
    for (uint64_t i = 0; i < n; ++i) {
        U256 x, y;
        memcpy(x.v, points + 8 * i, 32);
        memcpy(y.v, points + 8 * i + 4, 32);
        if (x.is_zero() && y.is_zero()) {
            out[2 * i] = x;
            out[2 * i + 1] = y;
            continue;
        }
        if (!(x < F.q) || !(y < F.q)) return fail(CW_EINVAL, what + "point " + std::to_string(i) + ": a coordinate is not below q");
        const U256 xm = mont ? x : F.to_mont(x), ym = mont ? y : F.to_mont(y);
        if (F.mont_mul(ym, ym) != F.addm(F.mont_mul(F.mont_mul(xm, xm), xm), three))
            return fail(CW_EINVAL, what + "point " + std::to_string(i) + " is not on the curve y^2 = x^3 + 3");
        out[2 * i] = xm;
        out[2 * i + 1] = ym;
    }
    return CW_OK;
}
// checked Montgomery images (g1_points_mont) to a new handle on `device`
static int g1_bases_upload(const std::vector<U256> &mont, int device, std::unique_ptr<cw_g1_bases> &out) {
    int rc = ensure_device(device);
    if (rc) return rc;
    auto b = std::make_unique<cw_g1_bases>();
    b->device = device;
    b->n = mont.size() / 2;
    if ((rc = upload(b->pts, mont.data(), (size_t)b->n * 64))) return rc;
    out = std::move(b);
    return CW_OK;
}

int cw_g1_bases_create(int prime_id, const uint64_t *points, uint64_t n, int device, cw_g1_bases **out) {
    if (!out || (!points && n)) return fail(CW_EINVAL, "null argument");
    *out = nullptr;
    if (prime_id != CW_PRIME_BN128) return fail(CW_EINVAL, "G1 bases are built for bn128 (BN254) only");
    if (n == 0 || n > MSM_MAX_N) return fail(CW_EINVAL, "the number of points must lie in [1, 2^26]");
    std::vector<U256> mont;
    int rc = g1_points_mont(points, n, false, "", mont);
    if (rc) return rc;
    std::unique_ptr<cw_g1_bases> b;
    if ((rc = g1_bases_upload(mont, device, b))) return rc;
    *out = b.release();
    return CW_OK;
}

void cw_g1_bases_destroy(cw_g1_bases *b) {
    if (!b) return;
    cudaSetDevice(b->device);
    delete b;
}

int cw_g1_msm_scratch_bytes(const cw_g1_bases *b, uint32_t count, uint64_t *bytes) {
    if (!b || !bytes || count == 0) return fail(CW_EINVAL, "bad argument");
    int rc = ensure_device(b->device);
    if (rc) return rc;
    MsmPlan p;
    if ((rc = msm_plan_for(b->n, count, p))) return rc;
    *bytes = p.total;
    return CW_OK;
}

// the argument checks of cw_g1_msm_batch / cw_g2_msm_batch that need no device; then the device pointers
static int msm_check_args(uint64_t n, const uint64_t *scalars_dev, uint64_t stride_elems, uint32_t count, uint64_t *out_dev,
                          void *scratch_dev) {
    if (!scalars_dev || !out_dev || !scratch_dev || count == 0) return fail(CW_EINVAL, "bad argument");
    if (stride_elems < n) return fail(CW_EINVAL, "stride_elems must be at least the number of points");
    if (((uintptr_t)scalars_dev | (uintptr_t)out_dev | (uintptr_t)scratch_dev) & 31u)
        return fail(CW_EINVAL, "device pointers must be 32-byte aligned");
    return CW_OK;
}
static int msm_check_pointers(int device, const uint64_t *scalars_dev, uint64_t *out_dev, void *scratch_dev) {
    for (const void *p : {(const void *)scalars_dev, (const void *)out_dev, (const void *)scratch_dev}) {
        cudaPointerAttributes a;
        if (cudaPointerGetAttributes(&a, p) != cudaSuccess) {
            cudaGetLastError();
            return fail(CW_EINVAL, "not a device pointer");
        }
        if (a.type != cudaMemoryTypeDevice && a.type != cudaMemoryTypeManaged) return fail(CW_EINVAL, "not device memory");
        if (a.device != device) return fail(CW_EINVAL, "device memory of another device than the bases'");
    }
    return CW_OK;
}

// the digits of instances [i0, i0 + cn) and their sort: sorted keys and values in the plan's keys[1] / vals[1].  The same
// for G1 and G2: the digits do not depend on the group.
static int msm_sorted_digits(const MsmPlan &p, char *S, const uint64_t *scalars_dev, uint64_t stride_elems, u32 n, u32 i0,
                             u32 cn, cudaStream_t st) {
    const u32 n_win = cn * p.W;
    const uint64_t N = (uint64_t)n_win * n;
    u32 *k0 = (u32 *)(S + p.keys[0]), *k1 = (u32 *)(S + p.keys[1]), *v0 = (u32 *)(S + p.vals[0]), *v1 = (u32 *)(S + p.vals[1]);
    msm_digits_kernel<<<grid_for(n, MSM_THREADS, 8, cn), MSM_THREADS, 0, st>>>((const uint4 *)(scalars_dev + 4 * (size_t)i0 * stride_elems),
                                                    stride_elems, n, p.c, p.W, cn, k0, v0);
    size_t cub_bytes = p.cub_bytes;
    CU(cub::DeviceRadixSort::SortPairs(S + p.cub, cub_bytes, k0, k1, v0, v1, (int)N, 0, (int)(p.c + msm_seg_bits(n_win)), st));
    return CW_OK;
}

int cw_g1_msm_batch(cw_g1_bases *b, const uint64_t *scalars_dev, uint64_t stride_elems, uint32_t count,
                    uint64_t *out_dev, void *scratch_dev, void *stream) {
    if (!b) return fail(CW_EINVAL, "bad argument");
    int rc = msm_check_args(b->n, scalars_dev, stride_elems, count, out_dev, scratch_dev);
    if (rc) return rc;
    if ((rc = ensure_device(b->device))) return rc;
    if ((rc = msm_check_pointers(b->device, scalars_dev, out_dev, scratch_dev))) return rc;
    MsmPlan p;
    if ((rc = msm_plan_for(b->n, count, p))) return rc;
    cudaStream_t st = (cudaStream_t)stream;
    char *S = (char *)scratch_dev;
    const u32 n = (u32)b->n;
    const u32 m = p.B < MSM_SEG ? p.B : MSM_SEG, per = p.B / m;
    for (u32 i0 = 0; i0 < count; i0 += p.chunk) {
        const u32 cn = std::min(p.chunk, count - i0), n_win = cn * p.W;
        const uint64_t N = (uint64_t)n_win * n;
        if ((rc = msm_sorted_digits(p, S, scalars_dev, stride_elems, n, i0, cn, st))) return rc;
        const u32 *k1 = (const u32 *)(S + p.keys[1]), *v1 = (const u32 *)(S + p.vals[1]);
        Xyzz *buckets = (Xyzz *)(S + p.buckets);
        CU(cudaMemsetAsync(buckets, 0, (size_t)n_win * p.B * sizeof(Xyzz), st));
        // level 0 over the sorted affine items, then levels over the partial sums until one thread covered a level
        uint64_t threads = (N + MSM_RUN - 1) / MSM_RUN, items = N;
        int lv = 0;
        msm_runs_kernel<true><<<(u32)((threads + MSM_THREADS - 1) / MSM_THREADS), MSM_THREADS, 0, st>>>(
            k1, v1, b->pts.get(), nullptr, N, p.c, buckets, (u32 *)(S + p.lv_keys[0]), (Xyzz *)(S + p.lv_pts[0]));
        while (threads > 1) {
            items = msm_level_out(items);
            threads = (items + MSM_RUN - 1) / MSM_RUN;
            msm_runs_kernel<false><<<(u32)((threads + MSM_THREADS - 1) / MSM_THREADS), MSM_THREADS, 0, st>>>(
                (const u32 *)(S + p.lv_keys[lv]), nullptr, nullptr, (const Xyzz *)(S + p.lv_pts[lv]), items, p.c, buckets,
                (u32 *)(S + p.lv_keys[lv ^ 1]), (Xyzz *)(S + p.lv_pts[lv ^ 1]));
            lv ^= 1;
        }
        Xyzz *segs = (Xyzz *)(S + p.segs), *wins = (Xyzz *)(S + p.wins);
        const uint64_t seg_threads = (uint64_t)n_win * per;
        msm_segments_kernel<<<(u32)((seg_threads + MSM_THREADS - 1) / MSM_THREADS), MSM_THREADS, 0, st>>>(buckets, p.B, n_win, segs);
        msm_windows_kernel<<<n_win, MSM_THREADS, 0, st>>>(segs, per, wins);
        msm_final_kernel<<<(cn + MSM_THREADS - 1) / MSM_THREADS, MSM_THREADS, 0, st>>>(wins, p.W, p.c, cn,
                                                                                      (uint4 *)(out_dev + 8 * (size_t)i0));
        CU(cudaGetLastError());
    }
    return CW_OK;
}

// ---- multi-scalar multiplication on G2 of BN254 (msm_g2.cuh, kernels in msm_g2.cu) ------------------------------------
struct cw_g2_bases {
    int device = 0;
    uint64_t n = 0;
    DevPtr<u32> pts;   // [n][32] u32: Montgomery x.c0, x.c1, y.c0, y.c1; all zeros = infinity
};

// b' = 3 / (9 + u), canonical (c0, c1)
static const uint64_t G2_TWIST_B[2][4] = {
    {0x3267e6dc24a138e5ull, 0xb5b4c5e559dbefa3ull, 0x81be18991be06ac3ull, 0x2b149d40ceb8aaaeull},
    {0xe4a2bd0685c315d2ull, 0xa74fa084e52d1852ull, 0xcd2cafadeed8fdf4ull, 0x009713b03af0fed4ull},
};

// n affine G2 points [n][2][2][4] u64, canonical or Montgomery images (`mont`), checked as g1_points_mont does: all zeros
// is infinity, anything else has its four coefficients below q and lies on E'
static int g2_points_mont(const uint64_t *points, uint64_t n, bool mont, const std::string &what, std::vector<U256> &out) {
    const FieldParams F = make_field(MSM_PRIME);
    // Fq2 on the host, Montgomery images (c0, c1): the check y^2 = x^3 + b' is written apart from the device formulas
    struct E2 { U256 c0, c1; };
    auto mul = [&](const E2 &a, const E2 &b) {
        const U256 t0 = F.mont_mul(a.c0, b.c0), t1 = F.mont_mul(a.c1, b.c1);
        const U256 m = F.mont_mul(F.addm(a.c0, a.c1), F.addm(b.c0, b.c1));
        return E2{F.subm(t0, t1), F.subm(F.subm(m, t0), t1)};
    };
    U256 b0, b1;
    memcpy(b0.v, G2_TWIST_B[0], 32);
    memcpy(b1.v, G2_TWIST_B[1], 32);
    const E2 bt{F.to_mont(b0), F.to_mont(b1)};
    out.assign(4 * n, U256());
    for (uint64_t i = 0; i < n; ++i) {
        U256 c[4];
        bool zero = true;
        for (int k = 0; k < 4; ++k) {
            memcpy(c[k].v, points + 16 * i + 4 * k, 32);
            zero = zero && c[k].is_zero();
        }
        if (zero) {
            for (int k = 0; k < 4; ++k) out[4 * i + k] = c[k];
            continue;
        }
        for (int k = 0; k < 4; ++k)
            if (!(c[k] < F.q))
                return fail(CW_EINVAL, what + "point " + std::to_string(i) + ": coefficient " + std::to_string(k) +
                                           " (x.c0, x.c1, y.c0, y.c1) is not below q");
        for (int k = 0; k < 4 && !mont; ++k) c[k] = F.to_mont(c[k]);
        const E2 x{c[0], c[1]}, y{c[2], c[3]};
        const E2 yy = mul(y, y), xxx = mul(mul(x, x), x);
        if (yy.c0 != F.addm(xxx.c0, bt.c0) || yy.c1 != F.addm(xxx.c1, bt.c1))
            return fail(CW_EINVAL, what + "point " + std::to_string(i) + " is not on the twist y^2 = x^3 + 3 / (9 + u)");
        for (int k = 0; k < 4; ++k) out[4 * i + k] = c[k];
    }
    return CW_OK;
}
static int g2_bases_upload(const std::vector<U256> &mont, int device, std::unique_ptr<cw_g2_bases> &out) {
    int rc = ensure_device(device);
    if (rc) return rc;
    auto b = std::make_unique<cw_g2_bases>();
    b->device = device;
    b->n = mont.size() / 4;
    if ((rc = upload(b->pts, mont.data(), (size_t)b->n * 128))) return rc;
    out = std::move(b);
    return CW_OK;
}

int cw_g2_bases_create(int prime_id, const uint64_t *points, uint64_t n, int device, cw_g2_bases **out) {
    if (!out || (!points && n)) return fail(CW_EINVAL, "null argument");
    *out = nullptr;
    if (prime_id != CW_PRIME_BN128) return fail(CW_EINVAL, "G2 bases are built for bn128 (BN254) only");
    if (n == 0 || n > MSM_MAX_N) return fail(CW_EINVAL, "the number of points must lie in [1, 2^26]");
    std::vector<U256> mont;
    int rc = g2_points_mont(points, n, false, "", mont);
    if (rc) return rc;
    std::unique_ptr<cw_g2_bases> b;
    if ((rc = g2_bases_upload(mont, device, b))) return rc;
    *out = b.release();
    return CW_OK;
}

void cw_g2_bases_destroy(cw_g2_bases *b) {
    if (!b) return;
    cudaSetDevice(b->device);
    delete b;
}

int cw_g2_msm_scratch_bytes(const cw_g2_bases *b, uint32_t count, uint64_t *bytes) {
    if (!b || !bytes || count == 0) return fail(CW_EINVAL, "bad argument");
    int rc = ensure_device(b->device);
    if (rc) return rc;
    MsmPlan p;
    if ((rc = msm_plan_for(b->n, count, p, MSM_G2_POINT_BYTES))) return rc;
    *bytes = p.total;
    return CW_OK;
}

int cw_g2_msm_batch(cw_g2_bases *b, const uint64_t *scalars_dev, uint64_t stride_elems, uint32_t count,
                    uint64_t *out_dev, void *scratch_dev, void *stream) {
    if (!b) return fail(CW_EINVAL, "bad argument");
    int rc = msm_check_args(b->n, scalars_dev, stride_elems, count, out_dev, scratch_dev);
    if (rc) return rc;
    if ((rc = ensure_device(b->device))) return rc;
    if ((rc = msm_check_pointers(b->device, scalars_dev, out_dev, scratch_dev))) return rc;
    MsmPlan p;
    if ((rc = msm_plan_for(b->n, count, p, MSM_G2_POINT_BYTES))) return rc;
    cudaStream_t st = (cudaStream_t)stream;
    char *S = (char *)scratch_dev;
    const u32 n = (u32)b->n;
    for (u32 i0 = 0; i0 < count; i0 += p.chunk) {
        const u32 cn = std::min(p.chunk, count - i0), n_win = cn * p.W;
        const uint64_t N = (uint64_t)n_win * n;
        if ((rc = msm_sorted_digits(p, S, scalars_dev, stride_elems, n, i0, cn, st))) return rc;
        void *buckets = S + p.buckets;
        CU(cudaMemsetAsync(buckets, 0, (size_t)n_win * p.B * MSM_G2_POINT_BYTES, st));
        // level 0 over the sorted affine items, then levels over the partial sums until one thread covered a level
        uint64_t threads = (N + MSM_RUN - 1) / MSM_RUN, items = N;
        int lv = 0;
        msm_g2_launch_runs(true, (const u32 *)(S + p.keys[1]), (const u32 *)(S + p.vals[1]), b->pts.get(), nullptr, N, p.c, buckets,
                           (u32 *)(S + p.lv_keys[0]), S + p.lv_pts[0], st);
        while (threads > 1) {
            items = msm_level_out(items);
            threads = (items + MSM_RUN - 1) / MSM_RUN;
            msm_g2_launch_runs(false, (const u32 *)(S + p.lv_keys[lv]), nullptr, nullptr, S + p.lv_pts[lv], items, p.c, buckets,
                               (u32 *)(S + p.lv_keys[lv ^ 1]), S + p.lv_pts[lv ^ 1], st);
            lv ^= 1;
        }
        msm_g2_launch_reduce(buckets, p.B, n_win, S + p.segs, S + p.wins, p.W, p.c, cn, (uint4 *)(out_dev + 16 * (size_t)i0), st);
        CU(cudaGetLastError());
    }
    return CW_OK;
}

// ---- multi-scalar multiplication on G1 of BLS12-381 (msm_bls12381.cuh, kernels in msm_bls12381.cu) -------------------
struct cw_bls12381_g1_bases {
    int device = 0;
    uint64_t n = 0;
    DevPtr<u32> pts;   // [n][24] u32: Montgomery x, y (12 limbs each); (0, 0) = infinity
};

int cw_bls12381_g1_bases_create(const uint64_t *points, uint64_t n, int device, cw_bls12381_g1_bases **out) {
    if (!out || (!points && n)) return fail(CW_EINVAL, "null argument");
    *out = nullptr;
    if (n == 0 || n > MSM_MAX_N) return fail(CW_EINVAL, "the number of points must lie in [1, 2^26]");
    std::vector<u32> mont(24 * n);
    for (uint64_t i = 0; i < n; ++i) {
        const int bad = bls12381_g1_point_mont(points + 12 * i, &mont[24 * i]);
        if (bad == 1) return fail(CW_EINVAL, "point " + std::to_string(i) + ": a coordinate is not below q");
        if (bad) return fail(CW_EINVAL, "point " + std::to_string(i) + " is not on the curve y^2 = x^3 + 4");
    }
    int rc = ensure_device(device);
    if (rc) return rc;
    auto b = std::make_unique<cw_bls12381_g1_bases>();
    b->device = device;
    b->n = n;
    if ((rc = upload(b->pts, mont.data(), mont.size() * 4))) return rc;
    *out = b.release();
    return CW_OK;
}

void cw_bls12381_g1_bases_destroy(cw_bls12381_g1_bases *b) {
    if (!b) return;
    cudaSetDevice(b->device);
    delete b;
}

int cw_bls12381_g1_msm_scratch_bytes(const cw_bls12381_g1_bases *b, uint32_t count, uint64_t *bytes) {
    if (!b || !bytes || count == 0) return fail(CW_EINVAL, "bad argument");
    int rc = ensure_device(b->device);
    if (rc) return rc;
    MsmPlan p;
    if ((rc = msm_plan_for(b->n, count, p, MSM_BLS_POINT_BYTES))) return rc;
    *bytes = p.total;
    return CW_OK;
}

int cw_bls12381_g1_msm_batch(cw_bls12381_g1_bases *b, const uint64_t *scalars_dev, uint64_t stride_elems, uint32_t count,
                             uint64_t *out_dev, void *scratch_dev, void *stream) {
    if (!b) return fail(CW_EINVAL, "bad argument");
    int rc = msm_check_args(b->n, scalars_dev, stride_elems, count, out_dev, scratch_dev);
    if (rc) return rc;
    if ((rc = ensure_device(b->device))) return rc;
    if ((rc = msm_check_pointers(b->device, scalars_dev, out_dev, scratch_dev))) return rc;
    MsmPlan p;
    if ((rc = msm_plan_for(b->n, count, p, MSM_BLS_POINT_BYTES))) return rc;
    cudaStream_t st = (cudaStream_t)stream;
    char *S = (char *)scratch_dev;
    const u32 n = (u32)b->n;
    for (u32 i0 = 0; i0 < count; i0 += p.chunk) {
        const u32 cn = std::min(p.chunk, count - i0), n_win = cn * p.W;
        const uint64_t N = (uint64_t)n_win * n;
        if ((rc = msm_sorted_digits(p, S, scalars_dev, stride_elems, n, i0, cn, st))) return rc;
        void *buckets = S + p.buckets;
        CU(cudaMemsetAsync(buckets, 0, (size_t)n_win * p.B * MSM_BLS_POINT_BYTES, st));
        // level 0 over the sorted affine items, then levels over the partial sums until one thread covered a level
        uint64_t threads = (N + MSM_RUN - 1) / MSM_RUN, items = N;
        int lv = 0;
        msm_bls12381_launch_runs(true, (const u32 *)(S + p.keys[1]), (const u32 *)(S + p.vals[1]), b->pts.get(), nullptr, N,
                                 p.c, buckets, (u32 *)(S + p.lv_keys[0]), S + p.lv_pts[0], st);
        while (threads > 1) {
            items = msm_level_out(items);
            threads = (items + MSM_RUN - 1) / MSM_RUN;
            msm_bls12381_launch_runs(false, (const u32 *)(S + p.lv_keys[lv]), nullptr, nullptr, S + p.lv_pts[lv], items, p.c,
                                     buckets, (u32 *)(S + p.lv_keys[lv ^ 1]), S + p.lv_pts[lv ^ 1], st);
            lv ^= 1;
        }
        msm_bls12381_launch_reduce(buckets, p.B, n_win, S + p.segs, S + p.wins, p.W, p.c, cn,
                                   (uint4 *)(out_dev + 12 * (size_t)i0), st);
        CU(cudaGetLastError());
    }
    return CW_OK;
}

// ---- multi-scalar multiplication on G2 of BLS12-381 (msm_bls12381_g2.cuh, kernels in msm_bls12381_g2.cu) ------------
struct cw_bls12381_g2_bases {
    int device = 0;
    uint64_t n = 0;
    DevPtr<u32> pts;   // [n][48] u32: Montgomery x.c0, x.c1, y.c0, y.c1 (12 limbs each); all zeros = infinity
};

int cw_bls12381_g2_bases_create(const uint64_t *points, uint64_t n, int device, cw_bls12381_g2_bases **out) {
    if (!out || (!points && n)) return fail(CW_EINVAL, "null argument");
    *out = nullptr;
    if (n == 0 || n > MSM_MAX_N) return fail(CW_EINVAL, "the number of points must lie in [1, 2^26]");
    std::vector<u32> mont(48 * n);
    for (uint64_t i = 0; i < n; ++i) {
        int coef = 0;
        const int bad = bls12381_g2_point_mont(points + 24 * i, &mont[48 * i], &coef);
        if (bad == 1)
            return fail(CW_EINVAL, "point " + std::to_string(i) + ": coefficient " + std::to_string(coef) +
                                       " (x.c0, x.c1, y.c0, y.c1) is not below q");
        if (bad) return fail(CW_EINVAL, "point " + std::to_string(i) + " is not on the twist y^2 = x^3 + 4 (1 + u)");
    }
    int rc = ensure_device(device);
    if (rc) return rc;
    auto b = std::make_unique<cw_bls12381_g2_bases>();
    b->device = device;
    b->n = n;
    if ((rc = upload(b->pts, mont.data(), mont.size() * 4))) return rc;
    *out = b.release();
    return CW_OK;
}

void cw_bls12381_g2_bases_destroy(cw_bls12381_g2_bases *b) {
    if (!b) return;
    cudaSetDevice(b->device);
    delete b;
}

int cw_bls12381_g2_msm_scratch_bytes(const cw_bls12381_g2_bases *b, uint32_t count, uint64_t *bytes) {
    if (!b || !bytes || count == 0) return fail(CW_EINVAL, "bad argument");
    int rc = ensure_device(b->device);
    if (rc) return rc;
    MsmPlan p;
    if ((rc = msm_plan_for(b->n, count, p, MSM_BLS_G2_POINT_BYTES))) return rc;
    *bytes = p.total;
    return CW_OK;
}

int cw_bls12381_g2_msm_batch(cw_bls12381_g2_bases *b, const uint64_t *scalars_dev, uint64_t stride_elems, uint32_t count,
                             uint64_t *out_dev, void *scratch_dev, void *stream) {
    if (!b) return fail(CW_EINVAL, "bad argument");
    int rc = msm_check_args(b->n, scalars_dev, stride_elems, count, out_dev, scratch_dev);
    if (rc) return rc;
    if ((rc = ensure_device(b->device))) return rc;
    if ((rc = msm_check_pointers(b->device, scalars_dev, out_dev, scratch_dev))) return rc;
    MsmPlan p;
    if ((rc = msm_plan_for(b->n, count, p, MSM_BLS_G2_POINT_BYTES))) return rc;
    cudaStream_t st = (cudaStream_t)stream;
    char *S = (char *)scratch_dev;
    const u32 n = (u32)b->n;
    for (u32 i0 = 0; i0 < count; i0 += p.chunk) {
        const u32 cn = std::min(p.chunk, count - i0), n_win = cn * p.W;
        const uint64_t N = (uint64_t)n_win * n;
        if ((rc = msm_sorted_digits(p, S, scalars_dev, stride_elems, n, i0, cn, st))) return rc;
        void *buckets = S + p.buckets;
        CU(cudaMemsetAsync(buckets, 0, (size_t)n_win * p.B * MSM_BLS_G2_POINT_BYTES, st));
        // level 0 over the sorted affine items, then levels over the partial sums until one thread covered a level
        uint64_t threads = (N + MSM_RUN - 1) / MSM_RUN, items = N;
        int lv = 0;
        msm_bls12381_g2_launch_runs(true, (const u32 *)(S + p.keys[1]), (const u32 *)(S + p.vals[1]), b->pts.get(), nullptr, N,
                                    p.c, buckets, (u32 *)(S + p.lv_keys[0]), S + p.lv_pts[0], st);
        while (threads > 1) {
            items = msm_level_out(items);
            threads = (items + MSM_RUN - 1) / MSM_RUN;
            msm_bls12381_g2_launch_runs(false, (const u32 *)(S + p.lv_keys[lv]), nullptr, nullptr, S + p.lv_pts[lv], items, p.c,
                                        buckets, (u32 *)(S + p.lv_keys[lv ^ 1]), S + p.lv_pts[lv ^ 1], st);
            lv ^= 1;
        }
        msm_bls12381_g2_launch_reduce(buckets, p.B, n_win, S + p.segs, S + p.wins, p.W, p.c, cn,
                                      (uint4 *)(out_dev + 24 * (size_t)i0), st);
        CU(cudaGetLastError());
    }
    return CW_OK;
}

// ---- Groth16 proofs: proving key (.zkey), prove calls, assembly (groth16.cuh, kernel in groth16.cu) -------------------
static const int G16_STAGES = 8;   // expansion, quotient, H, A, B1, B2, C, assembly

struct cw_groth16_key {
    int device = 0;
    uint64_t n_vars = 0, n_public = 0, log_n = 0, n_coefs = 0;
    uint64_t r1cs_digest = 0;                     // r1cs_digest of the R1CS the key was checked against
    std::unique_ptr<cw_g1_bases> A, B1, C, H;     // C: null when the circuit has no private signals (its term is infinity)
    std::unique_ptr<cw_g2_bases> B2;
    DevPtr<u32> consts;                           // Groth16Consts: alpha1, beta1, delta1, beta2, delta2 (Montgomery)
    std::vector<uint64_t> ic;                     // [n_public + 1][2][4] canonical: the verifier's IC points
    Event ev[G16_STAGES + 1];                     // stage boundaries of the last prove call (cw_groth16_last_ms)
    bool timed = false;
};

// stage boundaries: recorded on the prove call's stream, read by cw_groth16_last_ms
static int groth16_mark(cw_groth16_key *k, int stage, cudaStream_t st) {
    if (!k->ev[stage]) {
        int rc = make_event(k->ev[stage]);
        if (rc) return rc;
    }
    CU(cudaEventRecord(k->ev[stage].get(), st));
    return CW_OK;
}

// FNV-1a style hash over the words of the constraints (sizes, public counts, rows, wires, coefficient values): the
// identity a proving key is tied to.  Two loads of the same .r1cs have the same digest.
static uint64_t r1cs_digest(cw_r1cs *r) {
    std::lock_guard<std::mutex> lk(r->mu);
    if (r->digest) return r->digest;
    const R1csData &R = r->data;
    uint64_t h = 0xcbf29ce484222325ull;
    auto mix = [&](uint64_t w) { h = (h ^ w) * 0x100000001b3ull; };
    for (uint64_t w : {(uint64_t)R.prime_id, R.n_wires, R.n_constraints, (uint64_t)R.n_pub_out, (uint64_t)R.n_pub_in}) mix(w);
    for (uint64_t p : R.row_ptr) mix(p);
    for (size_t i = 0; i < R.col.size(); ++i) {
        mix(R.col[i]);
        for (int k = 0; k < 4; ++k) mix(R.dict[R.coef[i]].v[k]);
    }
    r->digest = h ? h : 1;
    return r->digest;
}

// grumpkin = BN254's base field q, bn128 = its scalar field r: the 32-byte fields section 2 of a BN254 .zkey carries
static const int ZKEY_Q_PRIME = CW_PRIME_GRUMPKIN, ZKEY_R_PRIME = CW_PRIME_BN128;

// the .zkey bytes, checked against the R1CS on the host; pointers into the caller's buffer
struct ZkeyView {
    const uint8_t *sec[10] = {};   // payload of sections 1..9 (index = id)
    uint64_t size[10] = {};
    uint32_t n_vars = 0, n_public = 0, domain = 0, n_coefs = 0;
};

static uint32_t le32(const uint8_t *p) { uint32_t v; memcpy(&v, p, 4); return v; }
static uint64_t le64(const uint8_t *p) { uint64_t v; memcpy(&v, p, 8); return v; }

static int zkey_parse(const uint8_t *z, size_t len, cw_r1cs *r, ZkeyView &v) {
    static const char *names[10] = {"", "header", "Groth16 header", "IC", "coefficients", "A", "B1", "B2", "C", "H"};
    auto sec = [&](int id) { return "section " + std::to_string(id) + " (" + names[id] + ")"; };
    if (len < 12 || memcmp(z, "zkey", 4) != 0) return fail(CW_EINVAL, "zkey: bad magic (not a .zkey file)");
    if (le32(z + 4) != 1) return fail(CW_EINVAL, "zkey: version " + std::to_string(le32(z + 4)) + ", expected 1");
    const uint32_t n_sections = le32(z + 8);
    uint64_t at = 12;
    for (uint32_t k = 0; k < n_sections; ++k) {
        if (len - at < 12) return fail(CW_EINVAL, "zkey: truncated: the header of section record " + std::to_string(k) + " lies past the end");
        const uint32_t id = le32(z + at);
        const uint64_t size = le64(z + at + 4);
        at += 12;
        if (size > len - at)
            return fail(CW_EINVAL, "zkey: truncated: section " + std::to_string(id) + " declares " + std::to_string(size) +
                                       " bytes, " + std::to_string(len - at) + " remain");
        if (id >= 1 && id <= 9) {
            if (v.sec[id]) return fail(CW_EINVAL, "zkey: duplicate " + sec((int)id));
            v.sec[id] = z + at;
            v.size[id] = size;
        }
        at += size;   // (section 10, the contributions, and unknown sections are skipped)
    }
    if (at != len) return fail(CW_EINVAL, "zkey: " + std::to_string(len - at) + " bytes after the last section");
    for (int id = 1; id <= 9; ++id)
        if (!v.sec[id]) return fail(CW_EINVAL, "zkey: missing " + sec(id));
    if (v.size[1] != 4) return fail(CW_EINVAL, "zkey: " + sec(1) + " has " + std::to_string(v.size[1]) + " bytes, expected 4");
    if (le32(v.sec[1]) != 1) return fail(CW_EINVAL, "zkey: protocol " + std::to_string(le32(v.sec[1])) + " is not Groth16 (1)");
    // section 2: n8q, q, n8r, r, nVars, nPublic, domainSize, alpha1, beta1, beta2, gamma2, delta1, delta2
    const uint8_t *h = v.sec[2];
    if (v.size[2] < 4) return fail(CW_EINVAL, "zkey: " + sec(2) + " is truncated");
    const uint32_t n8q = le32(h);
    if (n8q != 32) return fail(CW_EINVAL, "zkey: n8q = " + std::to_string(n8q) + ": only BN254 keys (32-byte fields) are read");
    const uint64_t h_size = 4 + 32 + 4 + 32 + 12 + 3 * 64 + 3 * 128;
    if (v.size[2] < 40) return fail(CW_EINVAL, "zkey: " + sec(2) + " is truncated");
    const uint32_t n8r = le32(h + 36);
    if (n8r != 32) return fail(CW_EINVAL, "zkey: n8r = " + std::to_string(n8r) + ": only BN254 keys (32-byte fields) are read");
    if (v.size[2] != h_size)
        return fail(CW_EINVAL, "zkey: " + sec(2) + " has " + std::to_string(v.size[2]) + " bytes, expected " + std::to_string(h_size));
    if (memcmp(h + 4, make_field(ZKEY_Q_PRIME).q.v, 32) != 0) return fail(CW_EINVAL, "zkey: q is not the BN254 base field");
    if (memcmp(h + 40, make_field(ZKEY_R_PRIME).q.v, 32) != 0) return fail(CW_EINVAL, "zkey: r is not the BN254 scalar field (bn128)");
    v.n_vars = le32(h + 72);
    v.n_public = le32(h + 76);
    v.domain = le32(h + 80);
    if (v.n_public >= v.n_vars)
        return fail(CW_EINVAL, "zkey: nPublic (" + std::to_string(v.n_public) + ") must be below nVars (" + std::to_string(v.n_vars) + ")");
    if (v.domain == 0 || (v.domain & (v.domain - 1)))
        return fail(CW_EINVAL, "zkey: domainSize " + std::to_string(v.domain) + " is not a power of two");
    if (v.size[4] < 4) return fail(CW_EINVAL, "zkey: " + sec(4) + " is truncated");
    v.n_coefs = le32(v.sec[4]);
    // the sizes the header implies, in 64-bit arithmetic (no count can wrap them)
    const uint64_t nv = v.n_vars, np = v.n_public;
    const uint64_t want[10] = {0, 4, h_size, (np + 1) * 64, 4 + (uint64_t)v.n_coefs * 44, nv * 64, nv * 64, nv * 128,
                               (nv - np - 1) * 64, (uint64_t)v.domain * 64};
    for (int id = 3; id <= 9; ++id)
        if (v.size[id] != want[id])
            return fail(CW_EINVAL, "zkey: " + sec(id) + " has " + std::to_string(v.size[id]) + " bytes, the header implies " +
                                       std::to_string(want[id]));
    // the key against the R1CS
    const R1csData &R = r->data;
    if (R.prime_id != CW_PRIME_BN128) return fail(CW_EINVAL, "zkey: the R1CS is not over bn128");
    if (nv != R.n_wires)
        return fail(CW_EINVAL, "zkey: nVars (" + std::to_string(nv) + ") differs from the R1CS's wires (" + std::to_string(R.n_wires) + ")");
    u32 log_n = 0, n_pub = 0;
    int rc = qap_domain(r, log_n, n_pub);
    if (rc) return rc;
    if (np != n_pub)
        return fail(CW_EINVAL, "zkey: nPublic (" + std::to_string(np) + ") differs from the R1CS's (" + std::to_string(n_pub) + ")");
    if ((uint64_t)v.domain != (1ull << log_n))
        return fail(CW_EINVAL, "zkey: domainSize " + std::to_string(v.domain) + " disagrees with the R1CS's domain 2^" + std::to_string(log_n));
    // section 4 as a multiset of (matrix, constraint, signal): the nonzero A and B terms of the R1CS and the rows
    // A[m + j][j] = 1, j <= nPublic.  The coefficient values are not compared: which form snarkjs stores them in (they
    // are scaled Montgomery images there) could not be confirmed against a file snarkjs wrote, and the quotient reads
    // A and B from the R1CS, so only the shape has to match.
    using Term = std::tuple<u32, uint64_t, u32>;
    std::vector<Term> want_t, got_t;
    const uint64_t m = R.n_constraints;
    for (uint64_t i = 0; i < m; ++i)
        for (u32 mat = 0; mat < 2; ++mat)
            for (uint64_t t = R.row_ptr[3 * i + mat]; t < R.row_ptr[3 * i + mat + 1]; ++t)
                if (!R.dict[R.coef[t]].is_zero()) want_t.emplace_back(mat, i, R.col[t]);
    for (uint64_t j = 0; j <= np; ++j) want_t.emplace_back(0u, m + j, (u32)j);
    got_t.reserve(v.n_coefs);
    for (uint64_t k = 0; k < v.n_coefs; ++k) {
        const uint8_t *e = v.sec[4] + 4 + 44 * k;
        got_t.emplace_back(le32(e), (uint64_t)le32(e + 4), le32(e + 8));
    }
    std::sort(want_t.begin(), want_t.end());
    std::sort(got_t.begin(), got_t.end());
    if (want_t != got_t)
        return fail(CW_EINVAL, "zkey: " + sec(4) + " lists " + std::to_string(got_t.size()) + " (matrix, constraint, signal) terms "
                               "that are not the R1CS's A and B terms (" + std::to_string(want_t.size()) + "): a key of another circuit");
    return CW_OK;
}

// cw_groth16_key_info / the handle: see include/circom_b200.h
int cw_groth16_key_create(const void *zkey, size_t len, const cw_r1cs *r_in, int device, cw_groth16_key **out) {
    if (!out || !zkey || !r_in) return fail(CW_EINVAL, "null argument");
    *out = nullptr;
    cw_r1cs *r = const_cast<cw_r1cs *>(r_in);   // (the digest is cached in the handle)
    ZkeyView v;
    int rc = zkey_parse((const uint8_t *)zkey, len, r, v);
    if (rc) return rc;
    const uint64_t nv = v.n_vars, np = v.n_public;
    if (nv > MSM_MAX_N || v.domain > MSM_MAX_N) return fail(CW_EINVAL, "zkey: more than 2^26 points in a base set");
    // every point on the host before any device is touched
    const uint8_t *h = v.sec[2] + 84;   // alpha1 +0, beta1 +64, beta2 +128, gamma2 +256, delta1 +384, delta2 +448
    std::vector<U256> g1c, g2c, ic, a, b1, c, hh, b2;
    std::vector<uint64_t> buf(3 * 8);
    memcpy(buf.data(), h, 64);              // alpha1
    memcpy(buf.data() + 8, h + 64, 64);     // beta1
    memcpy(buf.data() + 16, h + 384, 64);   // delta1
    if ((rc = g1_points_mont(buf.data(), 3, true, "zkey: section 2 (alpha1, beta1, delta1): ", g1c))) return rc;
    buf.assign(3 * 16, 0);
    memcpy(buf.data(), h + 128, 128);       // beta2
    memcpy(buf.data() + 16, h + 256, 128);  // gamma2 (checked; the prover does not use it)
    memcpy(buf.data() + 32, h + 448, 128);  // delta2
    if ((rc = g2_points_mont(buf.data(), 3, true, "zkey: section 2 (beta2, gamma2, delta2): ", g2c))) return rc;
    auto words = [](const uint8_t *p, uint64_t n_u64) {
        std::vector<uint64_t> w(n_u64);
        memcpy(w.data(), p, n_u64 * 8);
        return w;
    };
    if ((rc = g1_points_mont(words(v.sec[3], (np + 1) * 8).data(), np + 1, true, "zkey: section 3 (IC): ", ic))) return rc;
    if ((rc = g1_points_mont(words(v.sec[5], nv * 8).data(), nv, true, "zkey: section 5 (A): ", a))) return rc;
    if ((rc = g1_points_mont(words(v.sec[6], nv * 8).data(), nv, true, "zkey: section 6 (B1): ", b1))) return rc;
    if ((rc = g2_points_mont(words(v.sec[7], nv * 16).data(), nv, true, "zkey: section 7 (B2): ", b2))) return rc;
    if ((rc = g1_points_mont(words(v.sec[8], (nv - np - 1) * 8).data(), nv - np - 1, true, "zkey: section 8 (C): ", c))) return rc;
    if ((rc = g1_points_mont(words(v.sec[9], (uint64_t)v.domain * 8).data(), v.domain, true, "zkey: section 9 (H): ", hh))) return rc;
    auto k = std::make_unique<cw_groth16_key>();
    k->device = device;
    k->n_vars = nv;
    k->n_public = np;
    k->n_coefs = v.n_coefs;
    while ((1ull << k->log_n) < v.domain) ++k->log_n;
    k->r1cs_digest = r1cs_digest(r);
    const FieldParams F = make_field(MSM_PRIME);
    k->ic.resize(ic.size() * 4);
    for (size_t i = 0; i < ic.size(); ++i) {
        const U256 cv = ic[i].is_zero() ? ic[i] : F.from_mont(ic[i]);   // ((0, 0) stays (0, 0): from_mont(0) = 0)
        memcpy(k->ic.data() + 4 * i, cv.v, 32);
    }
    std::vector<U256> cs;   // Groth16Consts order: alpha1, beta1, delta1, beta2, delta2
    cs.insert(cs.end(), g1c.begin(), g1c.end());
    cs.insert(cs.end(), g2c.begin(), g2c.begin() + 4);
    cs.insert(cs.end(), g2c.begin() + 8, g2c.end());
    static_assert(G16_CONSTS_WORDS == 14 * 8, "Groth16Consts layout: 3 G1 and 2 G2 points");
    if ((rc = g1_bases_upload(a, device, k->A))) return rc;   // (the first device call: ensure_device)
    if ((rc = g1_bases_upload(b1, device, k->B1))) return rc;
    if (nv - np - 1 && (rc = g1_bases_upload(c, device, k->C))) return rc;
    if ((rc = g1_bases_upload(hh, device, k->H))) return rc;
    if ((rc = g2_bases_upload(b2, device, k->B2))) return rc;
    if ((rc = upload(k->consts, cs.data(), cs.size() * 32))) return rc;
    *out = k.release();
    return CW_OK;
}

void cw_groth16_key_destroy(cw_groth16_key *k) {
    if (!k) return;
    cudaSetDevice(k->device);
    delete k;
}

int cw_groth16_key_info(const cw_groth16_key *k, uint64_t info[4]) {
    if (!k || !info) return fail(CW_EINVAL, "null argument");
    info[0] = k->n_vars;
    info[1] = k->n_public;
    info[2] = k->log_n;
    info[3] = k->n_coefs;
    return CW_OK;
}

int cw_groth16_key_ic(const cw_groth16_key *k, uint64_t *out) {
    if (!k || !out) return fail(CW_EINVAL, "null argument");
    memcpy(out, k->ic.data(), k->ic.size() * 8);
    return CW_OK;
}

// the caller's scratch: witness rows (cw_groth16_prove_batch only), h, the MSM results, (r, s), then one work area that
// the quotient uses first and every MSM after it (they run later on the same stream)
struct G16Layout {
    size_t rows = 0, h = 0, ma = 0, mb1 = 0, mc = 0, mh = 0, mb2 = 0, rs = 0, work = 0, total = 0;
};
static int groth16_layout(const cw_groth16_key *k, u32 count, G16Layout &L) {
    size_t at = 0;
    auto take = [&](size_t bytes) {
        const size_t o = at;
        at += (bytes + 255) & ~(size_t)255;
        return o;
    };
    const size_t n = (size_t)1 << k->log_n;
    L.rows = take((size_t)count * k->n_vars * 32);
    L.h = take((size_t)count * n * 32);
    L.ma = take((size_t)count * 64);
    L.mb1 = take((size_t)count * 64);
    L.mc = take((size_t)count * 64);
    L.mh = take((size_t)count * 64);
    L.mb2 = take((size_t)count * 128);
    L.rs = take((size_t)count * 64);
    uint64_t work = 2 * (uint64_t)count * n * 32, b = 0;
    int rc;
    for (const cw_g1_bases *g : {k->A.get(), k->B1.get(), k->C.get(), k->H.get()}) {
        if (!g) continue;
        if ((rc = cw_g1_msm_scratch_bytes(g, count, &b))) return rc;
        work = std::max(work, b);
    }
    if ((rc = cw_g2_msm_scratch_bytes(k->B2.get(), count, &b))) return rc;
    L.work = take(std::max(work, b));
    L.total = at;
    return CW_OK;
}

int cw_groth16_scratch_bytes(const cw_groth16_key *k, uint32_t count, uint64_t *bytes) {
    if (!k || !bytes || count == 0) return fail(CW_EINVAL, "bad argument");
    G16Layout L;
    int rc = groth16_layout(k, count, L);
    if (rc) return rc;
    *bytes = L.total;
    return CW_OK;
}

// (r, s) per proof: the caller's, checked to lie below r, or drawn from getrandom(2) by rejection below r
static int groth16_blinding(const uint64_t *rs, u32 count, std::vector<uint64_t> &out) {
    const U256 rr = make_field(CW_PRIME_BN128).q;
    out.assign((size_t)count * 8, 0);
    if (rs) {
        for (size_t i = 0; i < (size_t)count * 2; ++i) {
            U256 x;
            memcpy(x.v, rs + 4 * i, 32);
            if (!(x < rr))
                return fail(CW_EINVAL, std::string(i & 1 ? "s" : "r") + " of proof " + std::to_string(i / 2) + " is not below r");
        }
        memcpy(out.data(), rs, out.size() * 8);
        return CW_OK;
    }
    for (size_t i = 0; i < (size_t)count * 2; ++i) {
        U256 x;
        do {
            uint8_t *p = (uint8_t *)x.v;
            size_t got = 0;
            while (got < 32) {
                const ssize_t n = getrandom(p + got, 32 - got, 0);
                if (n < 0) {
                    if (errno == EINTR) continue;
                    return fail(CW_EIO, std::string("getrandom: ") + strerror(errno));
                }
                got += (size_t)n;
            }
            x.v[3] &= (1ull << 62) - 1;   // r < 2^254: keep 254 bits, accept below r
        } while (!(x < rr));
        memcpy(out.data() + 4 * i, x.v, 32);
    }
    return CW_OK;
}

// steps 3-6 on `st`: the MSMs over h and over the witness rows, then the assembly kernel
static int groth16_msms(cw_groth16_key *k, const uint64_t *rows, uint64_t stride, char *S, const G16Layout &L,
                        const std::vector<uint64_t> &rs, u32 count, uint64_t *proofs, cudaStream_t st) {
    auto at = [&](size_t off) { return (uint64_t *)(S + off); };
    void *work = S + L.work;
    CU(cudaMemcpyAsync(at(L.rs), rs.data(), rs.size() * 8, cudaMemcpyHostToDevice, st));   // (pageable: staged at once)
    int rc;
    if ((rc = cw_g1_msm_batch(k->H.get(), at(L.h), 1ull << k->log_n, count, at(L.mh), work, st))) return rc;
    if ((rc = groth16_mark(k, 3, st))) return rc;
    if ((rc = cw_g1_msm_batch(k->A.get(), rows, stride, count, at(L.ma), work, st))) return rc;
    if ((rc = groth16_mark(k, 4, st))) return rc;
    if ((rc = cw_g1_msm_batch(k->B1.get(), rows, stride, count, at(L.mb1), work, st))) return rc;
    if ((rc = groth16_mark(k, 5, st))) return rc;
    if ((rc = cw_g2_msm_batch(k->B2.get(), rows, stride, count, at(L.mb2), work, st))) return rc;
    if ((rc = groth16_mark(k, 6, st))) return rc;
    if (k->C) {
        if ((rc = cw_g1_msm_batch(k->C.get(), rows + 4 * (k->n_public + 1), stride, count, at(L.mc), work, st))) return rc;
    } else {
        CU(cudaMemsetAsync(at(L.mc), 0, (size_t)count * 64, st));   // no private signals: the C term is infinity
    }
    if ((rc = groth16_mark(k, 7, st))) return rc;
    groth16_launch_assemble(k->consts.get(), at(L.ma), at(L.mb1), at(L.mb2), at(L.mc), at(L.mh), at(L.rs), count, proofs, st);
    CU(cudaGetLastError());
    if ((rc = groth16_mark(k, 8, st))) return rc;
    k->timed = true;
    return CW_OK;
}

static int groth16_check_r1cs(const cw_groth16_key *k, cw_r1cs *r) {
    if (r1cs_digest(r) != k->r1cs_digest) return fail(CW_EINVAL, "the R1CS is not the one the proving key was checked against");
    return CW_OK;
}

int cw_groth16_prove_batch(cw_groth16_key *k, cw_r1cs *r, cw_batch *b, uint32_t first, uint32_t count, const uint64_t *rs,
                           uint64_t *proofs_dev, void *scratch_dev) {
    if (!k || !r || !b || count == 0 || (uint64_t)first + count > b->batch) return fail(CW_EINVAL, "bad argument");
    int rc = msm_check_args(0, (const uint64_t *)scratch_dev, 0, count, proofs_dev, scratch_dev);
    if (rc) return rc;
    if (!b->ran) return fail(CW_ESTATE, "batch has not been run");
    if ((rc = groth16_check_r1cs(k, r))) return rc;
    if (b->c->tape.n_witness != k->n_vars) return fail(CW_EINVAL, "the batch's witness size differs from the key's nVars");
    if (b->device != k->device) return fail(CW_EINVAL, "the batch and the proving key are on different devices");
    std::vector<uint64_t> rsv;
    if ((rc = groth16_blinding(rs, count, rsv))) return rc;
    if ((rc = ensure_device(k->device))) return rc;
    if ((rc = msm_check_pointers(k->device, (const uint64_t *)scratch_dev, proofs_dev, scratch_dev))) return rc;
    G16Layout L;
    if ((rc = groth16_layout(k, count, L))) return rc;
    char *S = (char *)scratch_dev;
    uint64_t *rows = (uint64_t *)(S + L.rows);
    cudaStream_t st = b->stream.get();
    k->timed = false;
    if ((rc = groth16_mark(k, 0, st))) return rc;
    if ((rc = cw_batch_expand_witness(b, first, count, rows))) return rc;
    if ((rc = groth16_mark(k, 1, st))) return rc;
    if ((rc = cw_r1cs_quotient_batch(r, b, first, count, (uint64_t *)(S + L.h), (uint64_t *)(S + L.work)))) return rc;
    if ((rc = groth16_mark(k, 2, st))) return rc;
    return groth16_msms(k, rows, k->n_vars, S, L, rsv, count, proofs_dev, b->stream.get());
}

int cw_groth16_prove_strided(cw_groth16_key *k, cw_r1cs *r, const uint64_t *witness_dev, uint64_t stride_elems, uint32_t count,
                             const uint64_t *rs, uint64_t *proofs_dev, void *scratch_dev) {
    if (!k || !r || stride_elems >> 32) return fail(CW_EINVAL, "bad argument");
    int rc = msm_check_args(k->n_vars, witness_dev, stride_elems, count, proofs_dev, scratch_dev);
    if (rc) return rc;
    if ((rc = groth16_check_r1cs(k, r))) return rc;
    std::vector<uint64_t> rsv;
    if ((rc = groth16_blinding(rs, count, rsv))) return rc;
    if ((rc = ensure_device(k->device))) return rc;
    if ((rc = msm_check_pointers(k->device, witness_dev, proofs_dev, scratch_dev))) return rc;
    G16Layout L;
    if ((rc = groth16_layout(k, count, L))) return rc;
    char *S = (char *)scratch_dev;
    DevPtr<unsigned long long> fb_d;
    if ((rc = dev_alloc(fb_d, (size_t)count * 8))) return rc;
    k->timed = false;
    if ((rc = groth16_mark(k, 0, 0)) || (rc = groth16_mark(k, 1, 0))) return rc;   // (no expansion: the rows are given)
    if ((rc = quotient_on_store(r, k->device, nullptr, dense_store(witness_dev, stride_elems, count), 0, count,
                                (uint64_t *)(S + L.h), (uint64_t *)(S + L.work), fb_d.get(), 0)))
        return rc;
    if ((rc = groth16_mark(k, 2, 0))) return rc;
    if ((rc = groth16_msms(k, witness_dev, stride_elems, S, L, rsv, count, proofs_dev, 0))) return rc;
    CU(cudaStreamSynchronize(0));
    return CW_OK;
}

int cw_groth16_last_ms(cw_groth16_key *k, float ms[8]) {
    if (!k || !ms) return fail(CW_EINVAL, "null argument");
    if (!k->timed) return fail(CW_ESTATE, "no prove call has been issued on this key");
    CU(cudaSetDevice(k->device));
    CU(cudaEventSynchronize(k->ev[G16_STAGES].get()));
    for (int i = 0; i < G16_STAGES; ++i) CU(cudaEventElapsedTime(&ms[i], k->ev[i].get(), k->ev[i + 1].get()));
    return CW_OK;
}

int cw_groth16_proof_json(const uint64_t proof[32], char *out, size_t cap, size_t *len) {
    if (!proof) return fail(CW_EINVAL, "null argument");
    return copy_text(groth16_proof_json(proof), out, cap, len);
}

int cw_groth16_public_json(const uint64_t *public_signals, uint32_t n_public, char *out, size_t cap, size_t *len) {
    if (!public_signals && n_public) return fail(CW_EINVAL, "null argument");
    return copy_text(groth16_public_json(public_signals, n_public), out, cap, len);
}

// readWitness side of the file boundary: the 32-byte entries of a .wtns (written by this library, the reference
// calculator or snarkjs); out = NULL returns the count only
int cw_wtns_read(const char *path, int *prime_id, uint64_t *n_witness, uint64_t *out, size_t cap_entries) {
    if (!path || !n_witness) return fail(CW_EINVAL, "null argument");
    std::vector<uint64_t> w;
    int pid = 0;
    try {
        read_wtns(path, pid, w);
    } catch (const std::exception &e) {
        return fail(CW_EFORMAT, e.what());
    }
    if (prime_id) *prime_id = pid;
    *n_witness = w.size() / 4;
    if (!out) return CW_OK;
    if (cap_entries < w.size() / 4) return fail(CW_EINVAL, "buffer too small");
    memcpy(out, w.data(), w.size() * 8);
    return CW_OK;
}

// A.w o B.w == C.w for a .wtns file against a .r1cs file (what `snarkjs wtns check` does): first_bad = -1 if every
// constraint holds, else the smallest violated row
int cw_r1cs_check_files(const char *r1cs_path, const char *wtns_path, int device, int64_t *first_bad) {
    if (!r1cs_path || !wtns_path || !first_bad) return fail(CW_EINVAL, "null argument");
    cw_r1cs *loaded = nullptr;
    int rc = cw_r1cs_load(r1cs_path, &loaded);
    if (rc) return rc;
    std::unique_ptr<cw_r1cs, void (*)(cw_r1cs *)> r(loaded, cw_r1cs_destroy);
    std::vector<uint64_t> w;
    int pid = 0;
    try {
        read_wtns(wtns_path, pid, w);
    } catch (const std::exception &e) {
        return fail(CW_EFORMAT, e.what());
    }
    if (pid != r->data.prime_id || w.size() / 4 != r->data.n_wires)
        return fail(CW_EINVAL, "the witness and the constraint system do not match (prime or number of wires)");
    return cw_r1cs_check(r.get(), w.data(), 0, 1, device, first_bad, nullptr);
}

// ---- lowered circuit as a blob / multi-GPU plumbing -----------------------------------------------------------
int cw_circuit_serialize(const cw_circuit *c, uint8_t *out, size_t cap, size_t *len) {
    if (!c || !len) return fail(CW_EINVAL, "null argument");
    std::vector<uint8_t> blob;
    serialize_tape(c->tape, blob);
    *len = blob.size();
    if (!out) return CW_OK;
    if (cap < blob.size()) return fail(CW_EINVAL, "buffer too small");
    memcpy(out, blob.data(), blob.size());
    return CW_OK;
}

int cw_circuit_deserialize(const void *data, size_t len, cw_circuit **out) {
    if (!data || !out) return fail(CW_EINVAL, "null argument");
    auto c = std::make_unique<cw_circuit>();
    try {
        deserialize_tape((const uint8_t *)data, len, c->tape);
    } catch (const std::exception &e) {
        return fail(CW_EFORMAT, e.what());
    }
    *out = c.release();
    return CW_OK;
}

// packed records of instances [first, first + count) into caller-provided DEVICE memory (count * words * 4 bytes),
// asynchronously on the batch stream: what a gather to another GPU sends
int cw_batch_pack_device(cw_batch *b, uint32_t first, uint32_t count, uint32_t *dst_device) {
    if (!b || !dst_device || (uint64_t)first + count > b->batch) return fail(CW_EINVAL, "bad argument");
    if (!b->ran) return fail(CW_ESTATE, "batch has not been run");
    CU(cudaSetDevice(b->device));
    const PackLayout &L = b->c->pack_layout();
    return pack_rows(b, L, first, count, dst_device);
}

// NCCL is resolved at run time (dlopen): the library loads and every single-GPU entry point works on machines
// without NCCL, and inside a process that already carries a copy (PyTorch's) that copy is the one used.
namespace {
struct NcclApi {
    void *h = nullptr;
    ncclResult_t (*GetUniqueId)(ncclUniqueId *) = nullptr;
    ncclResult_t (*CommInitRank)(ncclComm_t *, int, ncclUniqueId, int) = nullptr;
    ncclResult_t (*CommDestroy)(ncclComm_t) = nullptr;
    ncclResult_t (*Broadcast)(const void *, void *, size_t, ncclDataType_t, int, ncclComm_t, cudaStream_t) = nullptr;
    ncclResult_t (*AllReduce)(const void *, void *, size_t, ncclDataType_t, ncclRedOp_t, ncclComm_t, cudaStream_t) = nullptr;
    ncclResult_t (*Send)(const void *, size_t, ncclDataType_t, int, ncclComm_t, cudaStream_t) = nullptr;
    ncclResult_t (*Recv)(void *, size_t, ncclDataType_t, int, ncclComm_t, cudaStream_t) = nullptr;
    ncclResult_t (*GroupStart)() = nullptr;
    ncclResult_t (*GroupEnd)() = nullptr;
    const char *(*GetErrorString)(ncclResult_t) = nullptr;
};
NcclApi g_nccl;
std::mutex g_nccl_mu;

int load_nccl() {
    std::lock_guard<std::mutex> lk(g_nccl_mu);
    if (g_nccl.h) return CW_OK;
    void *h = nullptr;
    const char *env = getenv("CW_NCCL_LIB");
    for (const char *name : {env ? env : "libnccl.so.2", "libnccl.so.2", "libnccl.so"}) {
        h = dlopen(name, RTLD_NOW | RTLD_GLOBAL);
        if (h) break;
    }
    if (!h) return fail(CW_ENODEV, "NCCL is not available (libnccl.so.2 could not be loaded)");
    NcclApi a;
    a.h = h;
#define CW_SYM(field, sym)                                             \
    *(void **)(&a.field) = dlsym(h, sym);                              \
    if (!a.field) return fail(CW_ENODEV, std::string("NCCL symbol missing: ") + sym)
    CW_SYM(GetUniqueId, "ncclGetUniqueId");
    CW_SYM(CommInitRank, "ncclCommInitRank");
    CW_SYM(CommDestroy, "ncclCommDestroy");
    CW_SYM(Broadcast, "ncclBroadcast");
    CW_SYM(AllReduce, "ncclAllReduce");
    CW_SYM(Send, "ncclSend");
    CW_SYM(Recv, "ncclRecv");
    CW_SYM(GroupStart, "ncclGroupStart");
    CW_SYM(GroupEnd, "ncclGroupEnd");
    CW_SYM(GetErrorString, "ncclGetErrorString");
#undef CW_SYM
    g_nccl = a;
    return CW_OK;
}
#define NC(call)                                                                                           \
    do {                                                                                                   \
        ncclResult_t r_ = (call);                                                                          \
        if (r_ != ncclSuccess) return fail(CW_ECUDA, std::string(#call) + ": " + g_nccl.GetErrorString(r_)); \
    } while (0)
}  // namespace

struct cw_comm {
    ncclComm_t comm = nullptr;
    int rank = 0, world = 1, device = 0;
    bool owned = false;
    Stream stream;
    uint64_t bytes_sent = 0, bytes_received = 0;  // payload bytes this rank moved through the data-path collectives
};

int cw_comm_unique_id(uint8_t id[CW_COMM_ID_BYTES]) {
    if (!id) return fail(CW_EINVAL, "null argument");
    int rc = load_nccl();
    if (rc) return rc;
    static_assert(sizeof(ncclUniqueId) == CW_COMM_ID_BYTES, "ncclUniqueId size");
    ncclUniqueId u;
    NC(g_nccl.GetUniqueId(&u));
    memcpy(id, &u, sizeof(u));
    return CW_OK;
}

int cw_comm_init(const uint8_t id[CW_COMM_ID_BYTES], int rank, int world, int device, cw_comm **out) {
    if (!id || !out || world < 1 || rank < 0 || rank >= world) return fail(CW_EINVAL, "bad argument");
    int rc = load_nccl();
    if (rc) return rc;
    if ((rc = ensure_device(device))) return rc;
    ncclUniqueId u;
    memcpy(&u, id, sizeof(u));
    auto c = std::make_unique<cw_comm>();
    c->rank = rank;
    c->world = world;
    c->device = device;
    if ((rc = make_stream(c->stream))) return rc;   // (before the communicator: nothing can fail after it exists)
    ncclResult_t r = g_nccl.CommInitRank(&c->comm, world, u, rank);
    if (r != ncclSuccess) return fail(CW_ECUDA, std::string("ncclCommInitRank: ") + g_nccl.GetErrorString(r));
    c->owned = true;
    *out = c.release();
    return CW_OK;
}

int cw_comm_from_nccl(void *nccl_comm, int rank, int world, int device, cw_comm **out) {
    if (!nccl_comm || !out || world < 1 || rank < 0 || rank >= world) return fail(CW_EINVAL, "bad argument");
    int rc = load_nccl();
    if (rc) return rc;
    if ((rc = ensure_device(device))) return rc;
    auto c = std::make_unique<cw_comm>();
    c->comm = (ncclComm_t)nccl_comm;
    c->rank = rank;
    c->world = world;
    c->device = device;
    if ((rc = make_stream(c->stream))) return rc;
    *out = c.release();
    return CW_OK;
}

void cw_comm_destroy(cw_comm *c) {
    if (!c) return;
    cudaSetDevice(c->device);
    if (c->stream) cudaStreamSynchronize(c->stream.get());
    if (c->owned && c->comm && g_nccl.CommDestroy) g_nccl.CommDestroy(c->comm);
    delete c;
}

int cw_comm_stats(const cw_comm *c, uint64_t *bytes_sent, uint64_t *bytes_received) {
    if (!c) return fail(CW_EINVAL, "null argument");
    if (bytes_sent) *bytes_sent = c->bytes_sent;
    if (bytes_received) *bytes_received = c->bytes_received;
    return CW_OK;
}

// The lowered circuit of `root` (instruction tape, constants, witness maps, function code, input tables, R1CS in
// CSR form) on every rank: ONE NCCL broadcast of the size and one of the blob; only the root lowers.
int cw_circuit_broadcast(cw_comm *cm, cw_circuit **c, int root) {
    if (!cm || !c || root < 0 || root >= cm->world) return fail(CW_EINVAL, "bad argument");
    if (cm->rank == root && !*c) return fail(CW_EINVAL, "the root must pass its circuit");
    CU(cudaSetDevice(cm->device));
    std::vector<uint8_t> blob;
    if (cm->rank == root) serialize_tape((*c)->tape, blob);
    unsigned long long n = blob.size();
    DevPtr<unsigned long long> n_d;
    int rc;
    if ((rc = upload(n_d, &n, 8))) return rc;
    NC(g_nccl.Broadcast(n_d.get(), n_d.get(), 8, ncclUint8, root, cm->comm, cm->stream.get()));
    CU(cudaStreamSynchronize(cm->stream.get()));
    CU(cudaMemcpy(&n, n_d.get(), 8, cudaMemcpyDeviceToHost));
    DevPtr<uint8_t> buf_d;
    if ((rc = dev_alloc(buf_d, n ? n : 16))) return rc;
    if (cm->rank == root) CU(cudaMemcpy(buf_d.get(), blob.data(), n, cudaMemcpyHostToDevice));
    NC(g_nccl.Broadcast(buf_d.get(), buf_d.get(), n, ncclUint8, root, cm->comm, cm->stream.get()));
    CU(cudaStreamSynchronize(cm->stream.get()));
    if (cm->rank == root) {
        cm->bytes_sent += n * (uint64_t)(cm->world - 1);
        return CW_OK;
    }
    blob.resize(n);
    CU(cudaMemcpy(blob.data(), buf_d.get(), n, cudaMemcpyDeviceToHost));
    rc = cw_circuit_deserialize(blob.data(), blob.size(), c);
    cm->bytes_received += n;
    return rc;
}

// Gather of witness vectors: every rank packs instances [first, first + count) of its batch on the device and sends
// the records to `root` over NVLink (grouped ncclSend / ncclRecv); on the root recv_device[r][count][words] holds
// rank r's records (its own are packed in place).  Packed records, not 32-byte rows: 30x fewer bytes for circuits
// of bit decompositions; the root expands what it needs (cw_circuit_pack_info).  ms = device time on the root /
// sender of pack + transfer.
int cw_batch_gather_witness_packed(cw_comm *cm, cw_batch *b, uint32_t first, uint32_t count, int root,
                                   uint32_t *recv_device, uint32_t *send_scratch_device, float *ms) {
    if (!cm || !b || root < 0 || root >= cm->world || (uint64_t)first + count > b->batch) return fail(CW_EINVAL, "bad argument");
    if (!b->ran) return fail(CW_ESTATE, "batch has not been run");
    if (cm->rank == root && !recv_device) return fail(CW_EINVAL, "the root needs a receive buffer");
    if (cm->rank != root && !send_scratch_device) return fail(CW_EINVAL, "senders need a scratch buffer of count * words * 4 bytes");
    CU(cudaSetDevice(b->device));
    const PackLayout &L = b->c->pack_layout();
    const size_t n = (size_t)count * L.words * 4;  // bytes per rank
    Event e0, e1;
    int rc;
    if ((rc = make_event(e0)) || (rc = make_event(e1))) return rc;
    CU(cudaEventRecord(e0.get(), b->stream.get()));
    uint32_t *mine = cm->rank == root ? recv_device + (size_t)root * count * L.words : send_scratch_device;
    if ((rc = cw_batch_pack_device(b, first, count, mine))) return rc;
    NC(g_nccl.GroupStart());
    if (cm->rank == root) {
        for (int r = 0; r < cm->world; ++r)
            if (r != root) NC(g_nccl.Recv(recv_device + (size_t)r * count * L.words, n, ncclUint8, r, cm->comm, b->stream.get()));
    } else {
        NC(g_nccl.Send(mine, n, ncclUint8, root, cm->comm, b->stream.get()));
    }
    NC(g_nccl.GroupEnd());
    CU(cudaEventRecord(e1.get(), b->stream.get()));
    CU(cudaStreamSynchronize(b->stream.get()));
    if (ms) CU(cudaEventElapsedTime(ms, e0.get(), e1.get()));
    if (cm->rank == root) cm->bytes_received += n * (uint64_t)(cm->world - 1);
    else cm->bytes_sent += n;
    return CW_OK;
}

// all ranks learn whether any instance of any rank failed: out[0] = number of instances with a failed assert,
// out[1] = number with a runtime error, summed over the communicator (ncclAllReduce of two counters)
int cw_status_allreduce(cw_comm *cm, cw_batch *b, uint64_t out[2]) {
    if (!cm || !b || !out) return fail(CW_EINVAL, "null argument");
    std::vector<int32_t> st(b->batch);
    int rc = cw_batch_status(b, st.data());
    if (rc) return rc;
    unsigned long long h[2] = {0, 0};
    for (int32_t s : st) {
        if (s > 0) ++h[0];
        else if (s < 0) ++h[1];
    }
    DevPtr<unsigned long long> d;
    if ((rc = dev_alloc(d, 16))) return rc;
    CU(cudaMemcpyAsync(d.get(), h, 16, cudaMemcpyHostToDevice, b->stream.get()));
    NC(g_nccl.AllReduce(d.get(), d.get(), 2, ncclUint64, ncclSum, cm->comm, b->stream.get()));
    CU(cudaMemcpyAsync(h, d.get(), 16, cudaMemcpyDeviceToHost, b->stream.get()));
    CU(cudaStreamSynchronize(b->stream.get()));
    out[0] = h[0];
    out[1] = h[1];
    return CW_OK;
}

// ---- field batch ops ---------------------------------------------------------------------------
int cw_fr_batch_op(int prime_id, int op, const uint64_t *a, const uint64_t *b, const uint64_t *c, uint64_t *r,
                   size_t n, int device) {
    if (!a || !r || prime_id < 0 || prime_id >= CW_N_PRIMES) return fail(CW_EINVAL, "bad argument");
    int rc = ensure_device(device);
    if (rc) return rc;
    DevPtr<uint4> A, B, C, Rr;
    DevPtr<int> err;
    if ((rc = upload(A, a, n * 32))) return rc;
    if (b && (rc = upload(B, b, n * 32))) return rc;
    if (c && (rc = upload(C, c, n * 32))) return rc;
    if ((rc = dev_alloc(Rr, n * 32 + 32))) return rc;
    if ((rc = dev_alloc(err, 4))) return rc;
    CU(cudaMemset(err.get(), 0, 4));
    with_prime(prime_id, [&](auto pr) {
        fr_batch_op_kernel<decltype(pr)::value><<<grid_for(n, 128, 16), 128>>>(op, A.get(), B.get(), C.get(), Rr.get(), n, err.get(),
                                                                               (u32)prime_id);
    });
    CU(cudaGetLastError());
    CU(cudaMemcpy(r, Rr.get(), n * 32, cudaMemcpyDeviceToHost));
    int herr = 0;
    CU(cudaMemcpy(&herr, err.get(), 4, cudaMemcpyDeviceToHost));
    return herr ? fail(CW_EINVAL, "division by zero in batch op") : CW_OK;
}

int cw_fr_mul_bench(int prime_id, size_t n, int iters, int device, float *ms) {
    if (prime_id < 0 || prime_id > 1 || !ms) return fail(CW_EINVAL, "the throughput probe is built for bn128 and bls12381");
    int rc = ensure_device(device);
    if (rc) return rc;
    std::vector<uint64_t> h(n * 4);
    uint64_t s = 0x9E3779B97F4A7C15ull;
    for (auto &x : h) {
        s ^= s << 13; s ^= s >> 7; s ^= s << 17;
        x = s;
    }
    for (size_t i = 0; i < n; ++i) h[4 * i + 3] &= 0x0FFFFFFFFFFFFFFFull;
    DevPtr<uint4> d;
    Event e0, e1;
    if ((rc = upload(d, h.data(), n * 32)) || (rc = make_event(e0)) || (rc = make_event(e1))) return rc;
    u32 grid = (u32)((n + 255) / 256);
    for (int rep = 0; rep < 2; ++rep) {
        CU(cudaEventRecord(e0.get()));
        with_prime(prime_id, [&](auto pr) {
            if constexpr (decltype(pr)::value >= 0) fr_mul_bench_kernel<decltype(pr)::value><<<grid, 256>>>(d.get(), n, iters);
        });
        CU(cudaEventRecord(e1.get()));
        CU(cudaEventSynchronize(e1.get()));
    }
    CU(cudaEventElapsedTime(ms, e0.get(), e1.get()));
    return CW_OK;
}

}  // extern "C"
