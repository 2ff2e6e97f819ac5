// TEST INFRASTRUCTURE: executes the lowered tape on the CPU with the very same field/ops source the
// kernels compile (circom_b200/csrc/fr_device.cuh is host+device code), so the lowering
// (flatten.cpp) and the device arithmetic can be checked against the oracle without a GPU.
// This is NOT a product code path: libcircom_b200.so has no CPU execution and tests that
// need real kernels are marked `gpu`.
#include <cstdio>
#include <cstring>
#include <string>
#include <vector>

#include "../../circom_b200/csrc/fr_device.cuh"
#include "../../circom_b200/csrc/tape.h"
#include "../../circom_b200/csrc/r1cs_small.h"
#include <algorithm>
#include <stdexcept>

using namespace cw;

static std::string g_err;

static unsigned long long g_narrow_calls = 0, g_wide_calls = 0;   // calls finished on the 128-bit / the full-width machine

extern "C" {
// counters of the two register machines since the last call (tests: the narrow one must actually run)
void hs_vm_counters(unsigned long long *narrow, unsigned long long *wide) {
    *narrow = g_narrow_calls;
    *wide = g_wide_calls;
    g_narrow_calls = g_wide_calls = 0;
}


const char *hs_last_error() { return g_err.c_str(); }

// ---- the compiled R1CS on the value store of an instance (emulation of r1cs_small_kernel + r1cs_check_kernel) ----
// Set up by hs_run_r1cs; called by hs_run when an instance has finished, with its slots and bit plane.
struct R1csHook {
    bool on = false;
    bool compiled = false;
    R1csCompiled C;
    int64_t tamper_wire = -1;       // this witness entry is overwritten in the store before the check
    U256 tamper_value;
    int64_t *first_bad_compiled = nullptr, *first_bad_plain = nullptr;   // per instance
    uint64_t n_small_rows = 0, n_wide_marks = 0, n_general_rows = 0;
};
static R1csHook g_hook;

static void r1cs_hook_instance(const Tape &t, std::vector<u32> &slots, std::vector<u32> &bitplane, uint32_t inst) {
    R1csHook &H = g_hook;
    const FieldParams &F = t.F;
    if (!H.compiled) {
        compile_r1cs_host(t.r1cs, F, &t, false, true, H.C);
        H.compiled = true;
        H.n_small_rows = H.C.perm_small.size();
        H.n_general_rows = H.C.perm.size();
    }
    auto value_at = [&](u32 loc) -> U256 {
        U256 v = u256_from_u64(0);
        if (loc & OPERAND_BIT) {
            const u32 pos = loc & OPERAND_BITPOS_MASK;
            v.v[0] = (bitplane[pos >> 5] >> (pos & 31u)) & 1u;
        } else memcpy(v.v, &slots[(size_t)loc * 8], 32);
        return v;
    };
    if (H.tamper_wire >= 0) {
        const u32 loc = t.witness_slot[(size_t)H.tamper_wire];
        if (loc & OPERAND_BIT) {
            const u32 pos = loc & OPERAND_BITPOS_MASK;
            bitplane[pos >> 5] = (bitplane[pos >> 5] & ~(1u << (pos & 31u))) | ((u32)(H.tamper_value.v[0] & 1u) << (pos & 31u));
        } else memcpy(&slots[(size_t)loc * 8], H.tamper_value.v, 32);
    }
    const R1csData &R = t.r1cs;
    // plain check on the dense witness row (the definition)
    int64_t plain = -1;
    {
        std::vector<U256> w(R.n_wires);
        for (uint64_t i = 0; i < R.n_wires; ++i) w[i] = value_at(t.witness_slot[i]);
        for (uint64_t row = 0; row < R.n_constraints && plain < 0; ++row) {
            U256 acc[3];
            for (int m = 0; m < 3; ++m) {
                acc[m] = u256_from_u64(0);
                for (uint64_t k = R.row_ptr[3 * row + m]; k < R.row_ptr[3 * row + m + 1]; ++k)
                    acc[m] = F.addm(acc[m], F.mulm(R.dict[R.coef[k]], w[R.col[k]]));
            }
            if (!(F.mulm(acc[0], acc[1]) == acc[2])) plain = (int64_t)row;
        }
    }
    // the compiled form
    uint64_t fb = ~0ull;
    auto general_row = [&](u32 row) {
        U256 acc[3];
        for (int m = 0; m < 3; ++m) {
            acc[m] = u256_from_u64(0);
            for (unsigned long long k = H.C.row_ptr[3 * (size_t)row + m]; k < H.C.row_ptr[3 * (size_t)row + m + 1]; ++k) {
                const R1csTerm &tm = H.C.terms[k];
                const u32 kd = tm.kind & 0xFFu, sh = (tm.kind >> 8) & 0xFFu;
                U256 x;
                bool neg = kd == 2 || kd == 4 || kd == 6;
                if (kd >= 5) {
                    const u32 first = (tm.kind >> 16) & 31u, cnt = ((tm.kind >> 21) & 31u) + 1u;
                    const u32 word = (bitplane[tm.loc] >> first) & (cnt >= 32u ? 0xFFFFFFFFu : ((1u << cnt) - 1u));
                    x = u256_from_u64(word);
                    for (u32 j = 0; j < sh; ++j) x = F.addm(x, x);
                } else {
                    x = value_at(tm.loc);
                    if (tm.brow != 0xFFFFFFFFu && !(x == u256_from_u64(0)) && !(x == u256_from_u64(1))) fb = std::min<uint64_t>(fb, tm.brow);
                    if (kd == 0) { x = F.mulm(R.dict[tm.coef], x); }
                    else if (kd >= 3) for (u32 j = 0; j < sh; ++j) x = F.addm(x, x);
                }
                acc[m] = neg ? F.subm(acc[m], x) : F.addm(acc[m], x);
            }
        }
        if (!(F.mulm(acc[0], acc[1]) == acc[2])) fb = std::min<uint64_t>(fb, row);
    };
    for (u32 row : H.C.perm) general_row(row);
    for (size_t k = 0; k < H.C.perm_small.size(); ++k) {     // as r1cs_small_kernel reads them: the grouped record list
        const u32 row = H.C.perm_small[k];
        const u32 base = H.C.sgroups[2 * (k >> 5)], counts = H.C.sgroups[2 * (k >> 5) + 1];
        size_t at = (size_t)base + (k & 31u);
        long long v[3];
        u32 wide = 0;
        for (int m = 0; m < 3; ++m) {
            const u32 n = (counts >> (8 * m)) & 0xFFu;
            unsigned long long pos = 0, neg = 0;
            for (u32 tt = 0; tt < n; ++tt, at += 32) {
                const R1csSmallRec rec = H.C.srecs[at];
                if (rec.loc & SM_RUN) r1cs_small_acc_run(pos, neg, rec.loc, rec.mag, bitplane[rec.loc & SM_LOC]);
                else if (rec.loc & SM_BIT) {
                    const u32 p = rec.loc & SM_BITPOS;
                    r1cs_small_acc(pos, neg, wide, rec.loc, rec.mag, (bitplane[p >> 5] >> (p & 31u)) & 1u, 0u);
                } else {
                    U256 x = value_at(rec.loc & OPERAND_SLOT_MASK);
                    const u32 upper = (u32)(x.v[0] >> 32) | (u32)x.v[1] | (u32)(x.v[1] >> 32) | (u32)x.v[2] | (u32)(x.v[2] >> 32) |
                                      (u32)x.v[3] | (u32)(x.v[3] >> 32);
                    if ((rec.loc & SM_BROW) && (upper || (u32)x.v[0] > 1u)) fb = std::min<uint64_t>(fb, H.C.sbrow[at]);
                    r1cs_small_acc(pos, neg, wide, rec.loc, rec.mag, (u32)x.v[0], upper);
                }
            }
            v[m] = (long long)(pos - neg);
        }
        if (wide) { ++H.n_wide_marks; general_row(row); }
        else if (!r1cs_small_holds(v[0], v[1], v[2])) fb = std::min<uint64_t>(fb, row);
    }
    for (size_t i = 0; i < H.C.bool_loc.size(); ++i) {
        U256 x = value_at(H.C.bool_loc[i]);
        if (!(x == u256_from_u64(0)) && !(x == u256_from_u64(1))) fb = std::min<uint64_t>(fb, H.C.bool_row[i]);
    }
    H.first_bad_compiled[inst] = fb == ~0ull ? -1 : (int64_t)fb;
    H.first_bad_plain[inst] = plain;
}


// returns 0 on success; witness[batch][W][4 u64]; status[batch] like cw_batch_status
// Model of the device interpreter: all ops of a level read first, then all results of the level are written
// (on the device the work items of a level run in any order between two barriers).  hs_check_levels proves that
// no level reads a slot it also writes, which makes every device order equivalent to this one - also when
// temporaries share slots (CW_FLAG_REUSE).
int hs_run(const uint8_t *cb2c, size_t len, uint32_t flags, const uint64_t *inputs, uint32_t batch,
           uint64_t *witness, int32_t *status, uint64_t *stats /*8*/) {
    Tape t;
    try {
        lower_circuit(cb2c, len, flags, t);
    } catch (const std::exception &e) {
        g_err = e.what();
        return -1;
    }
    FrParams P = make_dev_params(t.F);
    size_t n_ops = t.n_tape_ops();
    if (stats) {
        stats[0] = t.n_signals; stats[1] = n_ops; stats[2] = t.n_levels(); stats[3] = t.n_slots;
        stats[4] = t.n_mul_ops; stats[5] = t.n_conv_ops; stats[6] = t.r1cs.n_constraints; stats[7] = t.n_bitwords;
    }
    std::vector<u32> slots((size_t)t.n_slots * 8);
    std::vector<u32> bitplane(t.n_bitwords);   // CW_FLAG_BITPLANE tapes: one word per bit run
    std::vector<uint8_t> bit_written((size_t)t.n_bitwords * 32), slot_written(t.n_slots);
    for (uint32_t inst = 0; inst < batch; ++inst) {
        std::fill(slots.begin(), slots.end(), 0xDEADBEEFu);  // poison: reads before writes show up
        std::fill(bitplane.begin(), bitplane.end(), 0xDEADBEEFu);
        std::fill(bit_written.begin(), bit_written.end(), 0);
        std::fill(slot_written.begin(), slot_written.end(), 0);
        u32 one[8] = {1, 0, 0, 0, 0, 0, 0, 0};
        memcpy(&slots[0], one, 32);
        slot_written[0] = 1;
        for (uint64_t k = 0; k < t.n_inputs; ++k) {
            memcpy(&slots[(size_t)t.input_slot[k] * 8], inputs + ((size_t)inst * t.n_inputs + k) * 4, 32);
            slot_written[t.input_slot[k]] = 1;
        }
        uint32_t first_assert = 0xFFFFFFFFu;
        int err = 0;
        bool bad_read = false;
        auto operand = [&](u32 o, u32 *v) {
            if (o & OPERAND_CONST) { memcpy(v, t.consts[o & 0x7FFFFFFFu].v, 32); return; }
            if (o & OPERAND_BIT) {  // one bit of the bit plane
                const u32 pos = o & OPERAND_BITPOS_MASK;
                if ((pos >> 5) >= t.n_bitwords || !bit_written[pos]) bad_read = true;   // (reported below)
                memset(v, 0, 32);
                v[0] = (pos >> 5) < t.n_bitwords ? (bitplane[pos >> 5] >> (pos & 31u)) & 1u : 0u;
                return;
            }
            const u32 slot = o & OPERAND_SLOT_MASK;
            if (slot >= t.n_slots || !slot_written[slot]) { bad_read = true; memset(v, 0, 32); return; }
            memcpy(v, &slots[(size_t)slot * 8], 32);
        };
        std::vector<u32> results;   // results of one level: {dst, 8 words}
        std::vector<u32> bit_results;  // bit-plane words of one level: {word index, value, run length}
        for (size_t l = 0; l < t.n_levels(); ++l) {
            results.clear();
            bit_results.clear();
            auto put_slot = [&](u32 dst, const u32 *r) {
                results.push_back(dst);
                results.insert(results.end(), r, r + 8);
            };
            for (size_t item = t.level_start[l]; item < t.level_start[l + 1]; ++item) {
              u32 acc[2][8];   // the two accumulator registers of a fused work item
              bool acc_set[2] = {false, false};
              auto operand_acc = [&](u32 o, u32 *v) {
                  if (!(o & OPERAND_CONST) && (o & OPERAND_ACC)) {
                      if (!acc_set[o & 1u]) bad_read = true;
                      memcpy(v, acc[o & 1u], 32);
                      return;
                  }
                  operand(o, v);
              };
              for (size_t i = t.items[item]; i < t.items[item + 1]; ++i) {
                const uint32_t *opw = &t.ops[i * 4];
                const uint32_t op[4] = {opw[0] & 0xFFu, opw[1], opw[2], opw[3]};
                const uint32_t dst = opw[0] >> 8;
                u32 a[8], b[8], r[8];
                auto put = [&](u32 d_, const u32 *r_) {
                    if (d_ >= DST_ACC) { memcpy(acc[d_ - DST_ACC], r_, 32); acc_set[d_ - DST_ACC] = true; return; }
                    if (i + 1 != t.items[item + 1]) bad_read = true;   // only the last word of an item writes the store
                    put_slot(d_, r_);
                };
                if (op[0] == OP_CALL) {  // function call: one work item interprets the body
                    const uint32_t *ct = &t.call_tab[op[1]];
                    FnInfo fi{t.fn_info[ct[0] * 4], t.fn_info[ct[0] * 4 + 1], t.fn_info[ct[0] * 4 + 2], t.fn_info[ct[0] * 4 + 3]};
                    std::vector<u32> regs((size_t)VM_MAX_REGS * 8, 0);   // (frames of nested calls are stacked behind the first)
                    for (uint32_t k = 0; k < ct[1]; ++k) operand(ct[2 + k], &regs[(size_t)k * 8]);
                    int e = 0;
                    u32 ret_base, ret_cnt;
                    // as kernels.cuh exec_call: the 128-bit machine first, the full-width one when it gives up
                    static const bool vm_wide_env = getenv("CW_VM_WIDE") && atoi(getenv("CW_VM_WIDE"));
                    const bool vm_wide = vm_wide_env || t.F.qbits <= 128;   // (as capi.cu: the 128-bit machine needs a prime above 2^128)
                    const bool narrow = !vm_wide && vm_run_narrow(t.fn_code.data(), t.fn_info.data(), ct[0], regs.data(),
                                                                  (const u32 *)t.consts.data(), r, e, ret_base, ret_cnt);
                    g_narrow_calls += narrow;
                    g_wide_calls += !narrow;
                    if (!narrow) {
                        std::fill(regs.begin(), regs.end(), 0u);
                        for (uint32_t k = 0; k < ct[1]; ++k) operand(ct[2 + k], &regs[(size_t)k * 8]);
                        e = 0;
                        vm_run(t.fn_code.data(), t.fn_info.data(), ct[0], regs.data(), (const u32 *)t.consts.data(), r, P, e, ret_base,
                               ret_cnt);
                    }
                    const uint32_t *ex = ct + 2 + ct[1];
                    for (uint32_t k = 0; k < ex[0]; ++k) {   // results 1.. of `var q[k] = f(..)`
                        if (ex[1 + k] == 0xFFFFFFFFu) continue;
                        if (k + 1 >= ret_cnt) { e = 2; continue; }
                        u32 v[8];
                        vm_result(v, regs.data(), ret_base + k + 1, narrow);
                        put_slot(ex[1 + k], v);
                    }
                    if (e) err = 1;
                    put(dst, r);
                    continue;
                }
                operand_acc(op[1], a);
                operand_acc(op[2], b);
                if (op[0] == OP_BITS && (op[3] >> 24)) {  // run of single-bit extractions into consecutive slots
                    u32 run = (op[3] >> 24) + 1u, k = op[3] & 0xFFFFu;
                    if (t.n_bitwords) {  // the run is one word of the bit plane (dst = word index)
                        u32 word = 0;
                        for (u32 j = 0; j < run; ++j) {
                            u256_bits(r, a, (k + j) | (1u << 16));
                            word |= (r[0] & 1u) << j;
                        }
                        bit_results.push_back(dst);
                        bit_results.push_back(word);
                        bit_results.push_back(run);
                        continue;
                    }
                    for (u32 j = 0; j < run; ++j) {
                        u256_bits(r, a, (k + j) | (1u << 16));
                        put_slot(dst + j, r);
                    }
                    continue;
                }
                if (op[0] == OP_SELECT) {
                    u32 c[8];
                    operand(op[3], c);
                    memcpy(r, u256_is_zero(c) ? b : a, 32);
                } else if (op[0] == OP_ASSERT_EQ || op[0] == OP_ASSERT || op[0] == OP_ASSERT_BOOL || op[0] == OP_ASSERT_FITS) {
                    bool ok = op[0] == OP_ASSERT_EQ ? u256_eq(a, b) : op[0] == OP_ASSERT ? !u256_is_zero(a)
                              : op[0] == OP_ASSERT_BOOL ? (u256_is_zero(a) || u256_eq(a, b)) : (u256_bitlen(a) <= b[0]);
                    if (!ok && op[3] < first_assert) first_assert = op[3];
                    continue;
                } else {
                    fr_exec(op[0], r, a, b, op[3], P, err);
                }
                put(dst, r);
              }
            }
            for (size_t k = 0; k < results.size(); k += 9) {
                if (results[k] >= t.n_slots) { g_err = "destination out of range"; return -5; }
                memcpy(&slots[(size_t)results[k] * 8], &results[k + 1], 32);
                slot_written[results[k]] = 1;
            }
            for (size_t k = 0; k < bit_results.size(); k += 3) {
                if (bit_results[k] >= t.n_bitwords) { g_err = "bit-plane word out of range"; return -5; }
                bitplane[bit_results[k]] = bit_results[k + 1];
                for (u32 j = 0; j < bit_results[k + 2]; ++j) bit_written[(size_t)bit_results[k] * 32 + j] = 1;
            }
        }
        for (uint64_t w = 0; w < t.n_witness; ++w) {
            // without a bit plane witness_slot is the identity: slot w IS witness entry w
            u32 v[8];
            operand(t.witness_slot[w], v);
            memcpy(witness + ((size_t)inst * t.n_witness + w) * 4, v, 32);
        }
        if (bad_read) { g_err = "a slot or a bit of the bit plane was read before it was written (or is out of range)"; return -6; }
        if (g_hook.on) {
            try {
                r1cs_hook_instance(t, slots, bitplane, inst);
            } catch (const std::exception &e) {
                g_err = e.what();
                return -30;
            }
        }
        status[inst] = err ? -1 : (first_assert == 0xFFFFFFFFu ? 0 : (int32_t)(first_assert + 1));
    }
    return 0;
}

// hs_run + the compiled R1CS check on the value store each instance leaves (see r1cs_hook_instance).  tamper_wire >= 0:
// that witness entry is overwritten with tamper_value (4 x u64) before the check.  counters = {rows in perm_small, rows
// marked wide over all instances, rows in perm}.
int hs_run_r1cs(const uint8_t *cb2c, size_t len, uint32_t flags, const uint64_t *inputs, uint32_t batch, int64_t tamper_wire,
                const uint64_t *tamper_value, int64_t *first_bad_compiled, int64_t *first_bad_plain, uint64_t *counters) {
    Tape probe;
    try {
        lower_circuit(cb2c, len, flags, probe);
    } catch (const std::exception &e) {
        g_err = e.what();
        return -1;
    }
    std::vector<uint64_t> wit((size_t)batch * probe.n_witness * 4);
    std::vector<int32_t> st(batch);
    g_hook = R1csHook();
    g_hook.on = true;
    g_hook.tamper_wire = tamper_wire;
    if (tamper_value) memcpy(g_hook.tamper_value.v, tamper_value, 32);
    g_hook.first_bad_compiled = first_bad_compiled;
    g_hook.first_bad_plain = first_bad_plain;
    int rc = hs_run(cb2c, len, flags, inputs, batch, wit.data(), st.data(), nullptr);
    counters[0] = g_hook.n_small_rows;
    counters[1] = g_hook.n_wide_marks;
    counters[2] = g_hook.n_general_rows;
    g_hook = R1csHook();
    return rc;
}

// witness2SignalList of the lowered circuit; returns n_witness (or <0)
long hs_witness2signal(const uint8_t *cb2c, size_t len, uint32_t flags, uint64_t *out, size_t cap) {
    Tape t;
    try {
        lower_circuit(cb2c, len, flags, t);
    } catch (const std::exception &e) {
        g_err = e.what();
        return -1;
    }
    if (out && cap >= t.witness2signal.size()) memcpy(out, t.witness2signal.data(), t.witness2signal.size() * 8);
    return (long)t.witness2signal.size();
}

// Structure of the lowered tape:
//  * every operand was produced in an earlier level (and, with reused temporaries, the producer is the LATEST
//    writer of that slot before the reader's level - there is no other notion of "the right value" in the tape,
//    the value-level comparison against the evaluator in hs_run covers that);
//  * no level reads a slot that the same level writes, and no level writes a slot twice: between two barriers
//    the device runs the work items of a level in any order;
//  * witness-resident slots [0, n_resident) are written exactly once; only temporaries are recycled.
int hs_check_levels(const uint8_t *cb2c, size_t len, uint32_t flags) {
    Tape t;
    try {
        lower_circuit(cb2c, len, flags, t);
    } catch (const std::exception &e) {
        g_err = e.what();
        return -1;
    }
    if (t.items.empty() || t.items.back() != t.n_tape_ops() || (t.n_levels() && t.level_start[t.n_levels()] != t.n_items())) {
        g_err = "level / item tables do not cover the tape"; return -2;
    }
    for (size_t k = 0; k + 1 < t.items.size(); ++k)
        if (t.items[k] >= t.items[k + 1]) { g_err = "empty work item"; return -2; }
    const uint32_t n_res = (flags & 32u /* CW_FLAG_REUSE */) ? t.n_resident : t.n_slots;
    std::vector<uint32_t> def(t.n_slots, 0), writes(t.n_slots, 0), read_stamp(t.n_slots, 0), write_stamp(t.n_slots, 0);
    std::vector<uint32_t> bitlvl(t.n_bitwords, 0), bitrun(t.n_bitwords, 0);
    def[0] = 0xFFFFFFFFu;  // "written before the tape starts"
    writes[0]++;
    for (uint64_t k = 0; k < t.n_inputs; ++k) {
        if (t.input_slot[k] >= n_res) { g_err = "main input outside the resident slots"; return -8; }
        def[t.input_slot[k]] = 0xFFFFFFFFu;
        writes[t.input_slot[k]]++;
    }
    auto is_assert = [](uint32_t opc) { return opc == OP_ASSERT || opc == OP_ASSERT_EQ || opc == OP_ASSERT_BOOL || opc == OP_ASSERT_FITS; };
    for (size_t l = 0; l < t.n_levels(); ++l) {
        const uint32_t L = (uint32_t)l + 1;
        auto read = [&](uint32_t o) -> int {
            if (o & OPERAND_CONST) {
                if ((o & 0x7FFFFFFFu) >= t.consts.size()) { g_err = "constant index out of range"; return -3; }
                return 0;
            }
            if (o & OPERAND_BIT) {
                const uint32_t pos = o & OPERAND_BITPOS_MASK;
                if ((pos >> 5) >= t.n_bitwords || (pos & 31u) >= bitrun[pos >> 5] || !bitlvl[pos >> 5]) {
                    g_err = "bit operand out of range or not produced in an earlier level"; return -13;
                }
                return 0;
            }
            if (o & OPERAND_ACC) return 0;   // an accumulator of the same work item (checked by the item walk below)
            if (o & ~OPERAND_SLOT_MASK) { g_err = "unknown operand flag"; return -4; }
            if (o >= t.n_slots) { g_err = "slot out of range"; return -4; }
            if (!def[o]) { g_err = "operand not produced in an earlier level"; return -5; }
            read_stamp[o] = L;
            return 0;
        };
        // calls close their level (the kernel runs them in a loop of their own after the other work items)
        {
            bool seen_call = false;
            for (uint32_t item = t.level_start[l]; item < t.level_start[l + 1]; ++item) {
                const bool is_call = (t.ops[(size_t)t.items[item] * 4] & 0xFFu) == OP_CALL;
                if (is_call && t.items[item + 1] - t.items[item] != 1) { g_err = "a call shares its work item"; return -19; }
                if (!is_call && seen_call) { g_err = "a call is not at the end of its level"; return -19; }
                seen_call |= is_call;
            }
        }
        // reads of the level (definitions so far are all from earlier levels)
        // accumulator discipline inside a work item: written before read, only the last word writes the store
        for (uint32_t item = t.level_start[l]; item < t.level_start[l + 1]; ++item) {
            bool have[2] = {false, false};
            for (uint32_t i = t.items[item]; i < t.items[item + 1]; ++i) {
                const uint32_t *opw = &t.ops[(size_t)i * 4];
                const uint32_t opc = opw[0] & 0xFFu, dst = opw[0] >> 8;
                const bool last = i + 1 == t.items[item + 1];
                const bool c_imm = is_assert(opc) || opc == OP_BITS || opc == OP_BITSIP;
                if (opc != OP_CALL)
                    for (int k = 1; k <= 3; ++k) {
                        if (k == 3 && c_imm) break;
                        if (!(opw[k] & OPERAND_CONST) && (opw[k] & OPERAND_ACC) && !have[opw[k] & 1u]) { g_err = "accumulator read before it is written"; return -16; }
                    }
                if (!last) {
                    if (is_assert(opc) || dst < DST_ACC || opc == OP_CALL) { g_err = "inner word of a work item must write an accumulator"; return -17; }
                    have[dst - DST_ACC] = true;
                } else if (!is_assert(opc) && dst >= DST_ACC) { g_err = "last word of a work item writes an accumulator"; return -18; }
            }
        }
        for (uint32_t i = t.items[t.level_start[l]]; i < t.items[t.level_start[l + 1]]; ++i) {
            const uint32_t *opw = &t.ops[(size_t)i * 4];
            const uint32_t opc = opw[0] & 0xFFu;
            int rc;
            if (opc == OP_CALL) {
                const uint32_t *ct = &t.call_tab[opw[1]];
                for (uint32_t k = 0; k < ct[1]; ++k)
                    if ((rc = read(ct[2 + k]))) return rc;
                continue;
            }
            const bool c_imm = is_assert(opc) || opc == OP_BITS || opc == OP_BITSIP;
            for (int k = 1; k <= 3; ++k) {
                if (k == 3 && c_imm) break;
                if ((rc = read(opw[k]))) return rc;
            }
        }
        // writes of the level
        for (uint32_t i = t.items[t.level_start[l]]; i < t.items[t.level_start[l + 1]]; ++i) {
            const uint32_t *opw = &t.ops[(size_t)i * 4];
            const uint32_t opc = opw[0] & 0xFFu, dst = opw[0] >> 8;
            if (is_assert(opc) || dst >= DST_ACC) continue;
            const uint32_t run = opc == OP_BITS ? (opw[3] >> 24) + 1u : 1u;
            if (t.n_bitwords && run > 1) {  // bit plane: the run is word `dst`
                if (dst >= t.n_bitwords) { g_err = "bit-plane word out of range"; return -11; }
                if (bitrun[dst]) { g_err = "bit-plane word written twice"; return -12; }
                bitrun[dst] = run;
                continue;
            }
            auto write_one = [&](uint32_t s) -> int {
                if (s >= t.n_slots) { g_err = "destination out of range"; return -6; }
                if (read_stamp[s] == L) { g_err = "a level writes a slot that the same level reads"; return -14; }
                if (write_stamp[s] == L) { g_err = "a level writes a slot twice"; return -15; }
                write_stamp[s] = L;
                if (++writes[s] > 1 && s < n_res) { g_err = "slot written twice"; return -7; }
                return 0;
            };
            int rc;
            for (uint32_t j = 0; j < run; ++j)
                if ((rc = write_one(dst + j))) return rc;
            if (opc == OP_CALL) {  // the further results of the call
                const uint32_t *ex = &t.call_tab[opw[1]] + 2 + t.call_tab[opw[1] + 1];
                for (uint32_t k = 0; k < ex[0]; ++k)
                    if (ex[1 + k] != 0xFFFFFFFFu && (rc = write_one(ex[1 + k]))) return rc;
            }
        }
        for (uint32_t i = t.items[t.level_start[l]]; i < t.items[t.level_start[l + 1]]; ++i) {  // ... become visible after the barrier
            const uint32_t *opw = &t.ops[(size_t)i * 4];
            const uint32_t opc = opw[0] & 0xFFu, dst = opw[0] >> 8;
            if (is_assert(opc) || dst >= DST_ACC) continue;
            const uint32_t run = opc == OP_BITS ? (opw[3] >> 24) + 1u : 1u;
            if (t.n_bitwords && run > 1) { bitlvl[dst] = L; continue; }
            for (uint32_t j = 0; j < run; ++j) def[dst + j] = L;
            if (opc == OP_CALL) {
                const uint32_t *ex = &t.call_tab[opw[1]] + 2 + t.call_tab[opw[1] + 1];
                for (uint32_t k = 0; k < ex[0]; ++k)
                    if (ex[1 + k] != 0xFFFFFFFFu) def[ex[1 + k]] = L;
            }
        }
    }
    {   // every witness entry is produced exactly once, in a resident place, and no two entries share a place
        std::vector<uint8_t> seen_slot(t.n_slots, 0), seen_bit((size_t)t.n_bitwords * 32, 0);
        for (uint64_t w = 0; w < t.n_witness; ++w) {
            const uint32_t ws = t.witness_slot[w];
            if (ws & OPERAND_BIT) {
                const uint32_t pos = ws & OPERAND_BITPOS_MASK;
                if ((pos >> 5) >= t.n_bitwords || (pos & 31u) >= bitrun[pos >> 5] || seen_bit[pos]++) {
                    g_err = "witness entry maps to a bad bit-plane position"; return -8;
                }
            } else {
                if (ws >= n_res || writes[ws] != 1 || seen_slot[ws]++) { g_err = "witness slot not written exactly once"; return -8; }
            }
        }
    }
    return 0;
}

// single field op with the same representation handling as fr_batch_op_kernel
int hs_fr_op(int prime, int op, const uint64_t *A, const uint64_t *B, const uint64_t *C, uint64_t *R, size_t n) {
    FieldParams F = make_field(prime);
    FrParams P = make_dev_params(F);
    int any_err = 0;
    for (size_t i = 0; i < n; ++i) {
        u32 a[8], b[8] = {0}, c[8] = {0}, r[8];
        memcpy(a, A + 4 * i, 32);
        if (B) memcpy(b, B + 4 * i, 32);
        if (C) memcpy(c, C + 4 * i, 32);
        int e = 0;
        if (op == OP_MUL) {
            u32 am[8];
            fr_to_mont(am, a, P);
            fr_mont_mul(r, am, b, P);
        } else if (op == 2) {
            u32 bm[8], im[8];
            fr_to_mont(bm, b, P);
            fr_inv_mont(im, bm, P);
            fr_mont_mul(r, im, a, P);
        } else if (op == OP_POW) {
            u32 am[8], rm[8];
            fr_to_mont(am, a, P);
            fr_pow_mont(rm, am, b, P);
            fr_from_mont(r, rm, P);
        } else if (op == OP_INV) {
            u32 am[8], rm[8];
            fr_to_mont(am, a, P);
            fr_inv_mont(rm, am, P);
            fr_from_mont(r, rm, P);
        } else if (op == OP_SELECT) {
            memcpy(r, u256_is_zero(c) ? b : a, 32);
        } else {
            fr_exec((u32)op, r, a, b, 0, P, e);
        }
        any_err |= e;
        memcpy(R + 4 * i, r, 32);
    }
    return any_err;
}

// one operator of the 128-bit register machine (fr_device.cuh: vmn_apply); v = n x {a_lo, a_hi, b_lo, b_hi, c_lo, c_hi},
// out = n x {r_lo, r_hi}, ok[i] = 0 when the operator hands the call to the full-width machine
void hs_vmn_apply(int op, const uint64_t *v, uint64_t *out, uint8_t *ok, size_t n) {
    for (size_t i = 0; i < n; ++i) {
        N128 a{v[6 * i], v[6 * i + 1]}, b{v[6 * i + 2], v[6 * i + 3]}, c{v[6 * i + 4], v[6 * i + 5]}, r{0, 0};
        ok[i] = vmn_apply((u32)op, r, a, b, c) ? 1 : 0;
        out[2 * i] = r.lo;
        out[2 * i + 1] = r.hi;
    }
}

// R1CS check with the kernel's arithmetic (Montgomery coefficient dictionary)
int hs_r1cs_check(const uint8_t *cb2c, size_t len, const uint64_t *witness, uint32_t batch, int64_t *first_bad) {
    Tape t;
    try {
        lower_circuit(cb2c, len, 0, t);
    } catch (const std::exception &e) {
        g_err = e.what();
        return -1;
    }
    FrParams P = make_dev_params(t.F);
    const R1csData &R = t.r1cs;
    std::vector<U256> dm(R.dict.size());
    for (size_t i = 0; i < dm.size(); ++i) dm[i] = t.F.to_mont(R.dict[i]);
    for (uint32_t inst = 0; inst < batch; ++inst) {
        const uint64_t *w = witness + (size_t)inst * R.n_wires * 4;
        first_bad[inst] = -1;
        for (uint64_t row = 0; row < R.n_constraints && first_bad[inst] < 0; ++row) {
            u32 acc[3][8];
            for (int m = 0; m < 3; ++m) {
                u256_set_u32(acc[m], 0);
                for (uint64_t k = R.row_ptr[3 * row + m]; k < R.row_ptr[3 * row + m + 1]; ++k) {
                    u32 x[8], cm[8], p[8], s[8];
                    memcpy(x, w + 4 * (size_t)R.col[k], 32);
                    memcpy(cm, dm[R.coef[k]].v, 32);
                    fr_mont_mul(p, cm, x, P);
                    fr_add(s, acc[m], p, P);
                    memcpy(acc[m], s, 32);
                }
            }
            u32 ab[8], c1[8];
            fr_mont_mul(ab, acc[0], acc[1], P);
            fr_from_mont(c1, acc[2], P);
            if (!u256_eq(ab, c1)) first_bad[inst] = (int64_t)row;
        }
    }
    return 0;
}

// Census of the general-row terms the R1CS check compiles for the value layout of the lowered tape (r1cs_compile.cpp):
// out[0] runs of plane bits, out[1] runs at a shift above 80 (placed without the lazy 128-bit sum), out[2] runs with a
// negative coefficient, out[3] runs that start inside a plane word, out[4] runs of 32 bits at shift 96, out[5] terms
int hs_r1cs_term_census(const uint8_t *cb2c, size_t len, uint32_t flags, uint64_t *out) {
    Tape t;
    R1csCompiled C;
    try {
        lower_circuit(cb2c, len, flags, t);
        compile_r1cs_host(t.r1cs, t.F, &t, false, false, C);
    } catch (const std::exception &e) {
        g_err = e.what();
        return -1;
    }
    for (int i = 0; i < 6; ++i) out[i] = 0;
    for (const R1csTerm &tm : C.terms) {
        const u32 kd = tm.kind & 0xFFu, sh = (tm.kind >> 8) & 0xFFu, first = (tm.kind >> 16) & 31u, cnt = ((tm.kind >> 21) & 31u) + 1u;
        if (kd < 5u) continue;
        out[0] += 1;
        out[1] += sh > 80u;
        out[2] += kd == 6u;
        out[3] += first != 0u;
        out[4] += sh == 96u && cnt == 32u;
    }
    out[5] = C.terms.size();
    return 0;
}

int hs_write_r1cs(const uint8_t *cb2c, size_t len, const char *path) {
    Tape t;
    try {
        lower_circuit(cb2c, len, 0, t);
        write_r1cs(t.r1cs, t.F, path);
    } catch (const std::exception &e) {
        g_err = e.what();
        return -1;
    }
    return 0;
}

}  // extern "C"
