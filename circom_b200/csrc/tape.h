// Lowered circuit: the flat, levelised instruction tape + metadata + R1CS in CSR form.
#pragma once
#include <cstdint>
#include <string>
#include <vector>

#include "u256.h"
#include "r1cs_small.h"

namespace cw {

constexpr uint32_t OPERAND_CONST = 0x80000000u;  // operand bit31: index into the constant table
constexpr uint32_t OPERAND_SLOT_MASK = 0x00FFFFFFu;
// operand bit29 (tapes lowered with CW_FLAG_BITPLANE): the value is one bit of the instance's bit plane,
// bits 0-28 = word * 32 + bit.  witness_slot[] entries use the same encoding.
constexpr uint32_t OPERAND_BIT = 0x20000000u, OPERAND_BITPOS_MASK = 0x1FFFFFFFu;
// Fused work items: a work item is a short sequence of tape words (T.items delimits them) evaluated by one thread;
// all but the last write one of two accumulator registers instead of a slot (destination field DST_ACC + k) and later
// words of the same item read them (operand OPERAND_ACC | k).
constexpr uint32_t OPERAND_ACC = 0x10000000u, DST_ACC = 0x00FFFFFEu;
constexpr uint32_t WSLOT_MONT = 0x80000000u;     // witness_slot bit31: slot holds the Montgomery image
constexpr uint32_t NO_SLOT = 0xFFFFFFFFu;

struct InputInfo {
    std::string name;
    uint64_t hash;
    uint64_t signal_id;
    uint64_t size;
};

// same layout as HashSignalInfo (c_elements/common/circom.hpp:17-21)
struct HashEntry {
    uint64_t hash, signalid, signalsize;
};

struct R1csData {
    int prime_id = 0;
    uint64_t n_wires = 0;
    uint64_t n_constraints = 0;
    std::vector<uint64_t> row_ptr;  // 3*m+1 : row r of A at 3r, B at 3r+1, C at 3r+2
    std::vector<uint32_t> col;      // wire ids
    std::vector<uint32_t> coef;     // index into dict
    std::vector<U256> dict;         // distinct coefficients, canonical
    uint32_t n_pub_out = 0, n_pub_in = 0, n_prv_in = 0;
    // custom-gate sections 4 / 5 of a PLONK-style .r1cs (r1cs_writer.rs:356-454): carried through read -> write unchanged
    bool has_custom_gates = false;
    std::vector<std::pair<std::string, std::vector<U256>>> gates_used;        // (template name, parameters)
    std::vector<std::pair<uint32_t, std::vector<uint64_t>>> gates_applied;   // (index into gates_used, wires)
};

struct Tape {
    FieldParams F;
    uint32_t flags = 0;
    uint64_t n_signals = 0, n_witness = 0, n_inputs = 0, n_outputs = 0, n_components = 0;
    uint64_t n_ir_ops = 0, n_mul_ops = 0, n_conv_ops = 0, max_level_width = 0, n_asserts = 0;
    uint64_t slot_census[4] = {0, 0, 0, 0};  // value slots by static width: 1 bit, <= 32, <= 64 bits, wider
    // operators by emitted opcode (< 64) and the static width of their result and slot operands: <= 64, 128, 192 bits, wider
    uint64_t width_census[64 * 4] = {};
    uint64_t n_slot_operands = 0;  // operand reads of slots
    uint64_t n_stored = 0;         // values that reach the value store (slots / plane words written): n_values minus the fused ones
    uint64_t n_values = 0;         // values the tape computes per instance (every destination, each bit of a run)
    uint32_t n_resident = 0;  // slots [0, n_resident) hold witness entries for the whole run; the rest are reused temporaries (CW_FLAG_REUSE)
    uint32_t n_pre = 0;    // slot 0 = constant one, slots 1..n_inputs = main inputs
    uint32_t n_slots = 0;  // witness entries [0, n_witness) then the other values
    uint32_t n_bitwords = 0;  // 32-bit words of the bit plane per instance (0: every value is a 32-byte slot)
    std::vector<uint32_t> ops;          // 4 words per op: opcode | dst << 8, a, b, c
    std::vector<uint32_t> items;        // n_items + 1: work item k = tape words [items[k], items[k+1])
    std::vector<uint32_t> level_start;  // n_levels + 1, indexes work items
    std::vector<U256> consts;           // raw limb patterns (already in the form the consumer needs)
    std::vector<U256> dat_consts;       // the circuit's constant list as the .dat carries it (canonical; c_code_generator.rs:616-679)
    std::vector<uint32_t> witness_slot; // per witness entry (identity: witness entry i lives in slot i)
    std::vector<uint32_t> input_slot;   // slot of main input i
    // witness entries by static size class, for the packed device->host transfer
    std::vector<uint32_t> pk_bit_wire, pk_u64_wire, pk_full_wire;
    std::vector<uint8_t> wit_class;  // per witness entry: 0 bit, 1 <= 64 bits, 2 full
    std::vector<uint16_t> wit_bits;  // per witness entry: the canonical value is below 2^wit_bits (256: nothing known)
    // circom functions (data-dependent control flow): register-machine code, per-function
    // {code offset, n_instr, n_regs, n_params}, and the per-call tables {function, n_args, arg operands...}
    std::vector<uint32_t> fn_code, fn_info, call_tab;
    std::vector<uint64_t> witness2signal; // witness2SignalList (calcwit.hpp:54-56)
    std::vector<InputInfo> inputs;
    std::vector<HashEntry> hashmap;
    R1csData r1cs;
    // names of signals and components per template, when the description carries a symbols section (docs/CB2C.md):
    // the source of `.sym` (dag/src/sym_porting.rs).  Not part of the lowered-circuit blob.
    struct SymTemplate {
        uint32_t n_own = 0;
        uint64_t total_signals = 0;
        std::vector<uint32_t> subs;          // template of each sub-component
        std::vector<std::string> own, sub;   // names of the own signals / of the sub-components
    };
    // where each `===` / assert() of the description sits, in the numbering cw_batch_status reports: template instance and
    // first signal of the component that executes it (the reference prints the template name and the component trace,
    // c_code_generator.rs:461-468).  Not part of the lowered-circuit blob.
    // log() calls in execution order (LogBucket, log_bucket.rs:104-162): one record per argument - a string, a constant, or the
    // witness entry that holds the logged signal's value (an eliminated signal is read through the entry it was merged into)
    struct LogArg {
        uint8_t kind = 0;     // 0 string (idx into log_strings), 1 witness entry idx, 2 constant (idx into log_consts)
        uint8_t last = 0;     // last argument of its log() call: a newline follows
        uint32_t idx = 0;
    };
    std::vector<LogArg> log_args;
    std::vector<std::string> log_strings;
    std::vector<U256> log_consts;
    std::vector<uint32_t> assert_tid;
    std::vector<uint64_t> assert_start;
    std::vector<std::string> tmpl_names;
    std::vector<SymTemplate> sym;            // empty: no symbols
    // the compiler's io map (docs/CB2C.md, IOMP section), written into the `.dat` where the reference runtime looks for it
    // (c_code_generator.rs:681-735, main.cpp:57-93).  Not part of the lowered-circuit blob.
    struct IoDef {
        uint32_t offset = 0, size = 1, bus_id = 0;
        std::vector<uint32_t> lengths;
    };
    std::vector<std::pair<uint32_t, std::vector<IoDef>>> io_map;   // (template instance id, its signals), ascending ids
    uint32_t sym_main = 0;
    size_t n_tape_ops() const { return ops.size() / 4; }
    size_t n_items() const { return items.empty() ? 0 : items.size() - 1; }
    size_t n_levels() const { return level_start.empty() ? 0 : level_start.size() - 1; }
};

// The CSR of an R1CS compiled for one value layout (r1cs_compile.cpp): what the check kernels read.
struct R1csTerm {   // 16 bytes, read as one uint4 on the device
    uint32_t loc;    // location of the wire's value (slot id, or OPERAND_BIT | plane position; a plane word index for runs)
    uint32_t coef;   // coefficient dictionary index
    uint32_t kind;   // kind word (kernels.cuh: 0 general, 1/2 +-1, 3/4 +-2^k, 5/6 +- run of plane bits)
    uint32_t brow;   // boolean row x*(x-1) = 0 of this wire checked along with the term, or ~0
};
struct R1csCompiled {
    std::vector<unsigned long long> row_ptr;   // 3m + 1, into terms
    std::vector<R1csTerm> terms;
    std::vector<U256> dictM;                   // coefficient dictionary, Montgomery form
    std::vector<uint32_t> perm;                // general rows, sorted by structure
    std::vector<uint32_t> perm_small;          // rows small by shape (r1cs_small.h), sorted by structure
    // ... and their own term list: per group of 32 rows {first record, counts n0 | n1 << 8 | n2 << 16}; record t of row r of
    // group g at sgroups[2g] + t * 32 + r; sbrow (empty: no term carries one): the boolean row checked along with a record
    std::vector<uint32_t> sgroups;
    std::vector<struct R1csSmallRec> srecs;
    std::vector<uint32_t> sbrow;
    std::vector<uint32_t> bool_loc, bool_row;  // boolean rows no general row absorbs
    uint32_t mean_row_terms = 0;               // compiled terms per row of perm
    uint64_t n_terms = 0;
};
// T = the circuit whose value store the check reads (nullptr: dense witness rows, location = wire id).  Throws.
void compile_r1cs_host(const R1csData &R, const FieldParams &F, const Tape *T, bool no_bool_rows, bool want_small,
                       R1csCompiled &out);

// Parse a .cb2c description and lower it.  Throws std::runtime_error.
void lower_circuit(const uint8_t *data, size_t len, uint32_t flags, Tape &out);

uint64_t fnv1a(const char *s, size_t n);

// the lowered circuit as one blob (flatten.cpp): what rank 0 broadcasts, or an on-disk cache
void serialize_tape(const Tape &t, std::vector<uint8_t> &out);
void deserialize_tape(const uint8_t *data, size_t len, Tape &t);

// file formats (formats.cpp)
void write_r1cs(const R1csData &r, const FieldParams &F, const std::string &path);
void read_r1cs(const std::string &path, R1csData &out);
std::vector<uint8_t> wtns_bytes(const FieldParams &F, const uint64_t *witness, uint64_t n_witness);
size_t field_bytes(const FieldParams &F);   // element size in .r1cs / .wtns files: 32, or 8 for goldilocks
void write_dat(const Tape &t, const std::string &path);
// .wtns (main.cpp:288-334 / witness_calculator.js:212-276): returns the witness as 4 x u64 limbs per entry
void read_wtns(const std::string &path, int &prime_id, std::vector<uint64_t> &witness);
// .sym (constraint_writers/src/sym_writer.rs:4-38, dag/src/sym_porting.rs:16-33): one line per signal,
// `signal id,witness index or -1,node id,qualified name`.  Throws when the circuit carries no symbols.
void write_sym(const Tape &t, const std::string &path);
// the text the log() calls of the circuit print for one witness (n_witness x 4 u64), as the reference calculator prints it
std::string format_log(const Tape &t, const uint64_t *witness);
// snarkjs' proof.json of one proof ([32] u64: A x, y | B x.c0, x.c1, y.c0, y.c1 | C x, y, canonical; zeros = infinity) and
// public.json of n public signals ([n][4] u64 canonical), as compact JSON with decimal strings
std::string groth16_proof_json(const uint64_t *proof);
std::string groth16_public_json(const uint64_t *signals, uint32_t n);

}  // namespace cw
