// Byte-compatible file formats: .r1cs (read / write), .wtns (write), .dat (write).
#include <algorithm>
#include <cstdio>
#include <cstring>
#include <stdexcept>
#include <unordered_map>

#include "tape.h"

namespace cw {

namespace {
struct File {
    FILE *f;
    File(const std::string &p, const char *mode) : f(fopen(p.c_str(), mode)) {
        if (!f) throw std::runtime_error("cannot open " + p);
    }
    ~File() {
        if (f) fclose(f);
    }
    void w(const void *p, size_t n) {
        if (n && fwrite(p, 1, n, f) != n) throw std::runtime_error("write failed");
    }
    template <class T>
    void put(T v) {
        w(&v, sizeof(T));
    }
};

// minimal little-endian byte string of a wire id, as BigInt::to_bytes_le gives it
// (constraint_writers/src/r1cs_writer.rs:262-266); [0] for zero.
inline int le_len(uint32_t x) { return x >> 24 ? 4 : x >> 16 ? 3 : x >> 8 ? 2 : 1; }
inline bool wire_less(uint32_t a, uint32_t b) {
    int la = le_len(a), lb = le_len(b);
    for (int i = 0; i < std::min(la, lb); ++i) {
        uint8_t ba = (a >> (8 * i)) & 0xFF, bb = (b >> (8 * i)) & 0xFF;
        if (ba != bb) return ba < bb;
    }
    return la < lb;
}
}  // namespace

// bytes of one field element in files: whole 64-bit words of the prime (constraint_list/src/r1cs_porting.rs:6-10;
// 32 for the 256-bit primes, 8 for goldilocks - n8 of c_elements/common64/main.cpp:327)
size_t field_bytes(const FieldParams &F) { return (size_t)((F.qbits + 63) / 64) * 8; }

// Section order and header layout follow constraint_list/src/r1cs_porting.rs:19-53 and
// constraint_writers/src/r1cs_writer.rs:6-14,49-72,93-101,246-269,328-341.
void write_r1cs(const R1csData &r, const FieldParams &F, const std::string &path) {
    File f(path, "wb");
    f.w("r1cs", 4);
    f.put<uint32_t>(1);
    f.put<uint32_t>(r.has_custom_gates ? 5 : 3);
    // constraints section first
    uint64_t nnz = r.col.size();
    uint64_t m = r.n_constraints;
    const size_t fb = field_bytes(F);
    uint64_t csize = 3 * m * 4 + nnz * (4 + fb);
    f.put<uint32_t>(2);
    f.put<uint64_t>(csize);
    std::vector<uint32_t> order;
    for (uint64_t k = 0; k < 3 * m; ++k) {
        uint64_t b = r.row_ptr[k], e = r.row_ptr[k + 1];
        f.put<uint32_t>((uint32_t)(e - b));
        order.resize(e - b);
        for (uint64_t i = b; i < e; ++i) order[i - b] = (uint32_t)i;
        std::sort(order.begin(), order.end(), [&](uint32_t x, uint32_t y) { return wire_less(r.col[x], r.col[y]); });
        for (uint32_t i : order) {
            f.put<uint32_t>(r.col[i]);
            f.w(r.dict[r.coef[i]].v, fb);
        }
    }
    // header
    f.put<uint32_t>(1);
    f.put<uint64_t>(4 + fb + 4 * 4 + 8 + 4);
    f.put<uint32_t>((uint32_t)fb);
    f.w(F.q.v, fb);
    f.put<uint32_t>((uint32_t)r.n_wires);
    f.put<uint32_t>(r.n_pub_out);
    f.put<uint32_t>(r.n_pub_in);
    f.put<uint32_t>(r.n_prv_in);
    f.put<uint64_t>(r.n_wires);  // number of labels
    f.put<uint32_t>((uint32_t)m);
    // wire -> label map
    f.put<uint32_t>(3);
    f.put<uint64_t>(8 * r.n_wires);
    for (uint64_t i = 0; i < r.n_wires; ++i) f.put<uint64_t>(i);
    if (r.has_custom_gates) {
        // custom gates used (r1cs_writer.rs:356-392): u32 count; per gate: NUL-terminated name, u32 #parameters, field elements
        uint64_t sz = 4;
        for (auto &g : r.gates_used) sz += g.first.size() + 1 + 4 + fb * g.second.size();
        f.put<uint32_t>(4);
        f.put<uint64_t>(sz);
        f.put<uint32_t>((uint32_t)r.gates_used.size());
        for (auto &g : r.gates_used) {
            f.w(g.first.data(), g.first.size());
            f.put<uint8_t>(0);
            f.put<uint32_t>((uint32_t)g.second.size());
            for (const U256 &p : g.second) f.w(p.v, fb);
        }
        // custom gates applied (r1cs_writer.rs:408-440): u32 count; per application: u32 gate index, u32 #wires, u64 wires
        sz = 4;
        for (auto &a : r.gates_applied) sz += 8 + 8 * a.second.size();
        f.put<uint32_t>(5);
        f.put<uint64_t>(sz);
        f.put<uint32_t>((uint32_t)r.gates_applied.size());
        for (auto &a : r.gates_applied) {
            f.put<uint32_t>(a.first);
            f.put<uint32_t>((uint32_t)a.second.size());
            for (uint64_t w : a.second) f.put<uint64_t>(w);
        }
    }
}

void read_r1cs(const std::string &path, R1csData &out) {
    File f(path, "rb");
    fseek(f.f, 0, SEEK_END);
    long sz = ftell(f.f);
    fseek(f.f, 0, SEEK_SET);
    std::vector<uint8_t> buf(sz);
    if (sz && fread(buf.data(), 1, sz, f.f) != (size_t)sz) throw std::runtime_error("r1cs: read failed");
    auto need = [&](size_t off, size_t n) {
        if (n > buf.size() || off > buf.size() - n) throw std::runtime_error("r1cs: truncated file");  // (no wrap for n near 2^64)
    };
    auto u32 = [&](size_t off) { need(off, 4); uint32_t v; memcpy(&v, &buf[off], 4); return v; };
    auto u64 = [&](size_t off) { need(off, 8); uint64_t v; memcpy(&v, &buf[off], 8); return v; };
    need(0, 12);
    if (memcmp(buf.data(), "r1cs", 4)) throw std::runtime_error("r1cs: bad magic");
    if (u32(4) != 1) throw std::runtime_error("r1cs: unsupported version");
    uint32_t nsec = u32(8);
    size_t pos = 12, hdr = 0, cons = 0, hdr_len = 0, cons_len = 0, cgu = 0, cgu_len = 0, cga = 0, cga_len = 0;
    for (uint32_t s = 0; s < nsec; ++s) {
        uint32_t ty = u32(pos);
        uint64_t len = u64(pos + 4);
        pos += 12;
        need(pos, len);
        if (ty == 1) { hdr = pos; hdr_len = len; }
        if (ty == 2) { cons = pos; cons_len = len; }
        if (ty == 4) { cgu = pos; cgu_len = len; }
        if (ty == 5) { cga = pos; cga_len = len; }
        pos += len;
    }
    if (!hdr || !cons) throw std::runtime_error("r1cs: missing header or constraint section");
    need(hdr, 4);
    const uint32_t fs = u32(hdr);
    if ((fs != 32 && fs != 8) || hdr_len < 4 + (size_t)fs + 28) throw std::runtime_error("r1cs: only 32-byte and 8-byte fields are supported");
    need(hdr, 4 + (size_t)fs + 28);
    U256 q = u256_from_u64(0);
    memcpy(q.v, &buf[hdr + 4], fs);
    out.prime_id = prime_id_of(q);
    if (out.prime_id < 0 || field_bytes(make_field(out.prime_id)) != fs) throw std::runtime_error("r1cs: unsupported prime");
    size_t h = hdr + 4 + fs;
    out.n_wires = u32(h);
    out.n_pub_out = u32(h + 4);
    out.n_pub_in = u32(h + 8);
    out.n_prv_in = u32(h + 12);
    out.n_constraints = u32(h + 24);
    out.row_ptr.assign(1, 0);
    out.col.clear();
    out.coef.clear();
    out.dict.clear();
    std::unordered_map<std::string, uint32_t> idx;
    size_t p = cons, end = cons + cons_len;
    for (uint64_t k = 0; k < 3 * out.n_constraints; ++k) {
        if (p + 4 > end) throw std::runtime_error("r1cs: constraint section too short");
        uint32_t n = u32(p);
        p += 4;
        if ((uint64_t)n * (4 + fs) > end - p) throw std::runtime_error("r1cs: constraint section too short");
        size_t first = out.col.size();
        for (uint32_t j = 0; j < n; ++j) {
            uint32_t w = u32(p);
            if (w >= out.n_wires) throw std::runtime_error("r1cs: wire id out of range");
            std::string key((const char *)&buf[p + 4], fs);
            auto it = idx.find(key);
            uint32_t id;
            if (it == idx.end()) {
                U256 c = u256_from_u64(0);
                memcpy(c.v, key.data(), fs);
                // the check's arithmetic takes canonical coefficients (kinds by exact comparison with 2^k and q - 2^k)
                if (!(c < q)) throw std::runtime_error("r1cs: coefficient not reduced modulo the prime");
                id = (uint32_t)out.dict.size();
                out.dict.push_back(c);
                idx.emplace(std::move(key), id);
            } else id = it->second;
            out.col.push_back(w);
            out.coef.push_back(id);
            p += 4 + fs;
        }
        // numeric order inside the CSR row (files carry the byte-string order)
        std::vector<std::pair<uint32_t, uint32_t>> tmp;
        for (size_t i = first; i < out.col.size(); ++i) tmp.emplace_back(out.col[i], out.coef[i]);
        std::sort(tmp.begin(), tmp.end());
        for (size_t i = 0; i < tmp.size(); ++i) {
            out.col[first + i] = tmp[i].first;
            out.coef[first + i] = tmp[i].second;
        }
        out.row_ptr.push_back(out.col.size());
    }
    if (out.dict.empty()) out.dict.push_back(u256_from_u64(0));
    // custom-gate sections (r1cs_reader.rs:343-419): kept verbatim for the writer; the evaluator does not interpret them
    out.has_custom_gates = cgu != 0 || cga != 0;
    out.gates_used.clear();
    out.gates_applied.clear();
    if (cgu) {
        size_t q0 = cgu, qe = cgu + cgu_len;
        if (cgu_len < 4) throw std::runtime_error("r1cs: custom-gate section too short");
        uint32_t n = u32(q0);
        q0 += 4;
        for (uint32_t i = 0; i < n; ++i) {
            size_t z = q0;
            while (z < qe && buf[z]) ++z;
            if (z >= qe) throw std::runtime_error("r1cs: unterminated custom-gate name");
            std::string name((const char *)&buf[q0], z - q0);
            q0 = z + 1;
            if (q0 + 4 > qe) throw std::runtime_error("r1cs: custom-gate section too short");
            uint32_t np = u32(q0);
            q0 += 4;
            if ((uint64_t)np * fs > qe - q0) throw std::runtime_error("r1cs: custom-gate section too short");
            std::vector<U256> ps(np, u256_from_u64(0));
            for (uint32_t k = 0; k < np; ++k, q0 += fs) memcpy(ps[k].v, &buf[q0], fs);
            out.gates_used.emplace_back(std::move(name), std::move(ps));
        }
    }
    if (cga) {
        size_t q0 = cga, qe = cga + cga_len;
        if (cga_len < 4) throw std::runtime_error("r1cs: custom-gate section too short");
        uint32_t n = u32(q0);
        q0 += 4;
        for (uint32_t i = 0; i < n; ++i) {
            if (q0 + 8 > qe) throw std::runtime_error("r1cs: custom-gate section too short");
            uint32_t gi = u32(q0), ns = u32(q0 + 4);
            q0 += 8;
            if ((uint64_t)ns * 8 > qe - q0) throw std::runtime_error("r1cs: custom-gate section too short");
            if (gi >= out.gates_used.size()) throw std::runtime_error("r1cs: custom-gate application names an unknown gate");
            std::vector<uint64_t> ws(ns);
            for (uint32_t k = 0; k < ns; ++k, q0 += 8) ws[k] = u64(q0);
            out.gates_applied.emplace_back(gi, std::move(ws));
        }
    }
}

// .wtns: "wtns", u32 version 2, u32 2 sections; section 1 = {u32 n8 = 32, prime, u32 nVars}; section 2 = nVars x 32 bytes
void read_wtns(const std::string &path, int &prime_id, std::vector<uint64_t> &witness) {
    File f(path, "rb");
    fseek(f.f, 0, SEEK_END);
    long sz = ftell(f.f);
    fseek(f.f, 0, SEEK_SET);
    std::vector<uint8_t> buf(sz);
    if (sz && fread(buf.data(), 1, sz, f.f) != (size_t)sz) throw std::runtime_error("wtns: read failed");
    auto need = [&](size_t off, size_t n) {
        if (n > buf.size() || off > buf.size() - n) throw std::runtime_error("wtns: truncated file");
    };
    auto u32 = [&](size_t off) { need(off, 4); uint32_t v; memcpy(&v, &buf[off], 4); return v; };
    auto u64 = [&](size_t off) { need(off, 8); uint64_t v; memcpy(&v, &buf[off], 8); return v; };
    need(0, 12);
    if (memcmp(buf.data(), "wtns", 4)) throw std::runtime_error("wtns: bad magic");
    if (u32(4) != 2) throw std::runtime_error("wtns: unsupported version");
    uint32_t nsec = u32(8);
    size_t pos = 12, s1 = 0, s1_len = 0, s2 = 0, s2_len = 0;
    for (uint32_t s = 0; s < nsec; ++s) {
        uint32_t ty = u32(pos);
        uint64_t len = u64(pos + 4);
        pos += 12;
        need(pos, len);
        if (ty == 1) { s1 = pos; s1_len = len; }
        if (ty == 2) { s2 = pos; s2_len = len; }
        pos += len;
    }
    if (!s1 || !s2 || s1_len < 4 + 8 + 4) throw std::runtime_error("wtns: missing section");
    const uint32_t n8 = u32(s1);
    if ((n8 != 32 && n8 != 8) || s1_len < 4 + (size_t)n8 + 4) throw std::runtime_error("wtns: only 32-byte and 8-byte fields are supported");
    U256 q = u256_from_u64(0);
    memcpy(q.v, &buf[s1 + 4], n8);
    prime_id = prime_id_of(q);
    if (prime_id < 0 || field_bytes(make_field(prime_id)) != n8) throw std::runtime_error("wtns: unsupported prime");
    uint32_t n = u32(s1 + 4 + n8);
    if ((uint64_t)n * n8 != s2_len) throw std::runtime_error("wtns: witness section has the wrong size");
    witness.assign((size_t)n * 4, 0);   // always 4 x u64 per value in memory
    for (uint32_t i = 0; i < n; ++i) memcpy(&witness[(size_t)i * 4], &buf[s2 + (size_t)i * n8], n8);
    FieldParams F = make_field(prime_id);
    for (uint32_t i = 0; i < n; ++i) {
        U256 v;
        memcpy(v.v, &witness[(size_t)i * 4], 32);
        if (!(v < F.q)) throw std::runtime_error("wtns: value not reduced modulo the prime");
    }
}

// writeBinWitness (c_elements/common/main.cpp:288-334)
std::vector<uint8_t> wtns_bytes(const FieldParams &F, const uint64_t *witness, uint64_t n_witness) {
    const size_t n8 = field_bytes(F);
    std::vector<uint8_t> o(44 + n8 + n8 * n_witness);
    uint8_t *p = o.data();
    auto put32 = [&](uint32_t v) { memcpy(p, &v, 4); p += 4; };
    auto put64 = [&](uint64_t v) { memcpy(p, &v, 8); p += 8; };
    memcpy(p, "wtns", 4);
    p += 4;
    put32(2);
    put32(2);
    put32(1);
    put64(8 + n8);
    put32((uint32_t)n8);
    memcpy(p, F.q.v, n8);
    p += n8;
    put32((uint32_t)n_witness);
    put32(2);
    put64((uint64_t)n8 * n_witness);
    if (n8 == 32) memcpy(p, witness, 32 * n_witness);
    else for (uint64_t i = 0; i < n_witness; ++i) memcpy(p + i * n8, witness + 4 * i, n8);   // low words of the 4 x u64 values
    return o;
}

// generate_dat_file (c_code_generator.rs:818-865) for a circuit without run-time constants / io maps:
// the input hash map followed by the witness -> signal list.
void write_dat(const Tape &t, const std::string &path) {
    File f(path, "wb");
    for (const HashEntry &e : t.hashmap) {
        f.put<uint64_t>(e.hash);
        f.put<uint64_t>(e.signalid);
        f.put<uint64_t>(e.signalsize);
    }
    for (uint64_t i = 0; i < t.n_witness; ++i) f.put<uint64_t>(t.witness2signal[i]);
    // circuitConstants (generate_dat_constant_list, c_code_generator.rs:616-679): 40 bytes per constant -
    // {i32 shortVal, u32 type, n * R mod q}: values inside the signed 32-bit range carry shortVal and type
    // 0x40000000 (short + Montgomery), all others 0 and 0xC0000000 (long Montgomery).  The goldilocks runtime keeps its
    // constants as literals in the generated code: no constant list in its .dat (generate_dat_file, :838-841)
    for (const U256 &c : t.dat_consts) {
        if (field_bytes(t.F) == 8) break;
        U256 neg;
        u256_sub(neg, t.F.q, c);
        const bool is_neg = t.F.half < c;  // the signed view of generic/fr.cpp:1184-1218
        const U256 &mag = is_neg ? neg : c;
        const bool small = !(mag.v[1] | mag.v[2] | mag.v[3]) && (is_neg ? mag.v[0] <= 2147483648ull : mag.v[0] <= 2147483647ull);
        if (small) {
            f.put<int32_t>(is_neg ? (int32_t)(0 - (int64_t)mag.v[0]) : (int32_t)mag.v[0]);
            f.put<uint32_t>(0x40000000u);
        } else {
            f.put<int32_t>(0);
            f.put<uint32_t>(0xC0000000u);
        }
        U256 m = t.F.to_mont(c);
        f.w(m.v, 32);
    }
    // templateInsId2IOSignalInfo (generate_dat_io_signals_info, c_code_generator.rs:681-735; read back by loadCircuit,
    // main.cpp:57-93): the template ids, then per template {#signals, per signal: offset, #dimensions - 1, the dimensions
    // but the first, element size, bus id}, all u32.  The bus field map that follows (:737-794) has no entries: buses are
    // flattened by the producer.
    for (const auto &e : t.io_map) f.put<uint32_t>(e.first);
    for (const auto &e : t.io_map) {
        f.put<uint32_t>((uint32_t)e.second.size());
        for (const Tape::IoDef &d : e.second) {
            f.put<uint32_t>(d.offset);
            f.put<uint32_t>(d.lengths.empty() ? 0u : (uint32_t)d.lengths.size() - 1u);
            for (size_t i = 1; i < d.lengths.size(); ++i) f.put<uint32_t>(d.lengths[i]);
            f.put<uint32_t>(d.size);
            f.put<uint32_t>(d.bus_id);
        }
    }
}

// .sym: one line per signal, `signal id,witness index (-1: eliminated),node id,qualified name`, a component's own signals
// first, then its sub-components in creation order (visit_tree, dag/src/sym_porting.rs:16-33; the witness column as
// constraint_list/src/sym_porting.rs:24-31).  The node id is the DAG node of the component's template instance: the
// reference numbers nodes when their first instance finishes executing, children before parents - the post-order of
// first visits from main (the template order of a compiler-written description already is that order).  Signal 0, the
// constant one, has no line.
void write_sym(const Tape &t, const std::string &path) {
    if (t.sym.empty()) throw std::runtime_error("the circuit description carries no symbols section");
    std::vector<int64_t> wit(t.n_signals, -1);
    for (uint64_t i = 0; i < t.n_witness; ++i)
        if (t.witness2signal[i] < t.n_signals) wit[t.witness2signal[i]] = (int64_t)i;
    std::vector<int64_t> node(t.sym.size(), -1);
    {
        int64_t next = 0;
        std::vector<std::pair<uint32_t, size_t>> st;   // (template, next child)
        st.push_back({t.sym_main, 0});
        std::vector<uint8_t> open(t.sym.size(), 0);
        open[t.sym_main] = 1;
        while (!st.empty()) {
            auto &top = st.back();
            const Tape::SymTemplate &tt = t.sym[top.first];
            if (top.second < tt.subs.size()) {
                const uint32_t ch = tt.subs[top.second++];
                if (node[ch] < 0 && !open[ch]) { open[ch] = 1; st.push_back({ch, 0}); }
            } else {
                node[top.first] = next++;
                st.pop_back();
            }
        }
    }
    File f(path, "wb");
    std::string buf;
    buf.reserve(1u << 20);
    struct Frame { uint32_t tid; uint64_t start; std::string path; };
    std::vector<Frame> stack;
    stack.push_back({t.sym_main, 1, "main"});
    while (!stack.empty()) {
        Frame fr = std::move(stack.back());
        stack.pop_back();
        const Tape::SymTemplate &st = t.sym[fr.tid];
        if (fr.start + st.total_signals > t.n_signals) throw std::runtime_error("symbols do not match the circuit");
        for (uint32_t i = 0; i < st.n_own; ++i) {
            const uint64_t sig = fr.start + i;
            buf += std::to_string(sig);
            buf += ',';
            buf += std::to_string(wit[sig]);
            buf += ',';
            buf += std::to_string(node[fr.tid]);
            buf += ',';
            buf += fr.path;
            buf += '.';
            buf += st.own[i];
            buf += '\n';
            if (buf.size() > (1u << 20) - 8192) { f.w(buf.data(), buf.size()); buf.clear(); }
        }
        // children are visited in creation order: push them in reverse
        std::vector<uint64_t> starts(st.subs.size());
        uint64_t off = fr.start + st.n_own;
        for (size_t k = 0; k < st.subs.size(); ++k) { starts[k] = off; off += t.sym[st.subs[k]].total_signals; }
        for (size_t k = st.subs.size(); k-- > 0;) stack.push_back({st.subs[k], starts[k], fr.path + "." + st.sub[k]});
    }
    f.w(buf.data(), buf.size());
}

}  // namespace cw

namespace cw {
// decimal of a canonical 256-bit value, as Fr_element2str prints it (generic/fr.cpp:2836-2856: mpz_get_str base 10)
static std::string u256_decimal(const uint64_t *v) {
    uint32_t limb[8];
    for (int i = 0; i < 4; ++i) { limb[2 * i] = (uint32_t)v[i]; limb[2 * i + 1] = (uint32_t)(v[i] >> 32); }
    std::string out;
    for (;;) {
        uint64_t rem = 0;
        bool any = false;
        for (int i = 7; i >= 0; --i) {
            uint64_t cur = (rem << 32) | limb[i];
            limb[i] = (uint32_t)(cur / 1000000000u);
            rem = cur % 1000000000u;
            any |= limb[i] != 0;
        }
        char buf[16];
        snprintf(buf, sizeof(buf), any ? "%09u" : "%u", (unsigned)rem);
        out.insert(0, buf);
        if (!any) break;
    }
    return out;
}

static bool all_zero(const uint64_t *v, int n) {
    for (int i = 0; i < n; ++i)
        if (v[i]) return false;
    return true;
}

// snarkjs writes affine points in projective form [x, y, "1"]; the point at infinity is ["0", "1", "0"] in G1 and
// [["0", "0"], ["1", "0"], ["0", "0"]] in G2
std::string groth16_proof_json(const uint64_t *p) {
    auto d = [&](int k) { return "\"" + u256_decimal(p + 4 * k) + "\""; };
    auto g1 = [&](int k) {
        return all_zero(p + 4 * k, 8) ? std::string("[\"0\",\"1\",\"0\"]") : "[" + d(k) + "," + d(k + 1) + ",\"1\"]";
    };
    const std::string b = all_zero(p + 8, 16) ? std::string("[[\"0\",\"0\"],[\"1\",\"0\"],[\"0\",\"0\"]]")
                                              : "[[" + d(2) + "," + d(3) + "],[" + d(4) + "," + d(5) + "],[\"1\",\"0\"]]";
    return "{\"pi_a\":" + g1(0) + ",\"pi_b\":" + b + ",\"pi_c\":" + g1(6) + ",\"protocol\":\"groth16\",\"curve\":\"bn128\"}";
}

std::string groth16_public_json(const uint64_t *signals, uint32_t n) {
    std::string out = "[";
    for (uint32_t i = 0; i < n; ++i) out += (i ? ",\"" : "\"") + u256_decimal(signals + 4 * (size_t)i) + "\"";
    return out + "]";
}

// LogBucket (log_bucket.rs:104-162): the arguments of a call separated by one blank, values as decimals, a newline after the last
std::string format_log(const Tape &t, const uint64_t *witness) {
    std::string out;
    for (const Tape::LogArg &a : t.log_args) {
        if (a.kind == 0) out += t.log_strings[a.idx];
        else if (a.kind == 1) out += u256_decimal(witness + 4 * (size_t)a.idx);
        else out += u256_decimal(t.log_consts[a.idx].v);
        out += a.last ? "\n" : " ";
    }
    return out;
}
}  // namespace cw
