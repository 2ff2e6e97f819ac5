// Host half of the R1CS check: the CSR of a circuit compiled for one value layout (no CUDA here: the library uploads the
// result, tests/hostsim runs it on the CPU).
#include <algorithm>
#include <cstdlib>
#include <cstring>
#include <stdexcept>

#include "tape.h"
#include "r1cs_small.h"

namespace cw {

typedef uint32_t u32;

// Compile the CSR for one value layout: wire ids become locations (slot / plane bit; identity for dense witness
// rows), runs of plane bits with consecutive power-of-two coefficients become one term, boolean rows are absorbed
// or dropped where the storage makes them tautologies, rows are sorted by structure.  With `want_small`, rows whose
// terms are all small by shape (coefficients +-2^k, the bound of each of the three sums below 2^61 when every value is
// below 2^16) are listed apart (perm_small) with a term list of their own: the integer-row kernel decides them over the
// integers when the values it meets are small too (r1cs_small.h).
void compile_r1cs_host(const R1csData &R, const FieldParams &F, const Tape *T, bool no_bool_rows, bool want_small,
                       R1csCompiled &out) {
    if (T && T->n_witness != R.n_wires) throw std::runtime_error("the R1CS and the batch's circuit have different numbers of wires");
    auto loc_of = [&](u32 wire) -> u32 { return T ? T->witness_slot[wire] : wire; };
    // |a*b - c| must stay below q for the integer decision: every 256-bit prime, not goldilocks
    want_small = want_small && F.qbits > 130 && (T || R.n_wires <= OPERAND_SLOT_MASK);   // (locations of 24 bits in the records)
    std::vector<U256> &dm = out.dictM;
    dm.assign(R.dict.size(), u256_from_u64(0));
    std::vector<unsigned short> kind(R.dict.size());
    auto pow2_exp = [](const U256 &v) -> int {  // k if v == 2^k, else -1
        int k = -1;
        for (int i = 0; i < 256; ++i)
            if ((v.v[i >> 6] >> (i & 63)) & 1) {
                if (k >= 0) return -1;
                k = i;
            }
        return k;
    };
    for (size_t i = 0; i < R.dict.size(); ++i) {
        dm[i] = F.to_mont(R.dict[i]);
        U256 negv;
        u256_sub(negv, F.q, R.dict[i]);
        int kp = pow2_exp(R.dict[i]), kn = R.dict[i].is_zero() ? -1 : pow2_exp(negv);
        if (kp == 0) kind[i] = 1;
        else if (kn == 0) kind[i] = 2;
        else if (kp > 0 && kp < 250) kind[i] = (unsigned short)(3 | (kp << 8));
        else if (kn > 0 && kn < 250) kind[i] = (unsigned short)(4 | (kn << 8));
        else kind[i] = 0;
    }
    const size_t m = R.n_constraints;
    // boolean rows  x * (x - 1) = 0  (A = {x:1}, B = {x:1, one:-1}, C = {} or A/B swapped): they only need
    // `w[x] in {0,1}`.  A wire stored as one bit of the bit plane satisfies it by construction (the row is dropped);
    // otherwise the check rides on a term of a general row that reads the wire anyway, or goes to r1cs_bool_kernel.
    std::vector<u32> general, bool_wire, bool_row;
    auto is_unit = [&](uint64_t k, int want) { return (kind[R.coef[k]] & 0xFF) == want && (kind[R.coef[k]] >> 8) == 0; };
    for (size_t row = 0; row < m; ++row) {
        uint64_t p0 = R.row_ptr[3 * row], p1 = R.row_ptr[3 * row + 1], p2 = R.row_ptr[3 * row + 2], p3 = R.row_ptr[3 * row + 3];
        bool is_bool = false;
        u32 wire = 0;
        // (one block of one term, the other of two: three terms in A with B and C empty is A * 0 = 0, no boolean row)
        if (p3 == p2 && ((p1 - p0 == 1 && p2 - p1 == 2) || (p1 - p0 == 2 && p2 - p1 == 1))) {
            uint64_t s0 = (p1 - p0 == 1) ? p0 : p1, l0 = (p1 - p0 == 1) ? p1 : p0;  // single-term block / two-term block
            // two-term block is sorted by wire: {one: -1, x: +1}
            if (is_unit(s0, 1) && R.col[s0] != 0 && R.col[l0] == 0 && is_unit(l0, 2) && R.col[l0 + 1] == R.col[s0] && is_unit(l0 + 1, 1)) {
                is_bool = true;
                wire = R.col[s0];
            }
        }
        if (is_bool && !no_bool_rows) {
            if (loc_of(wire) & OPERAND_BIT) continue;  // a stored bit is 0 or 1
            bool_wire.push_back(wire);
            bool_row.push_back((u32)row);
        } else general.push_back((u32)row);
    }
    // compiled terms of the general rows
    std::vector<unsigned long long> &row_ptr = out.row_ptr;
    row_ptr.assign(3 * m + 1, 0);
    std::vector<uint8_t> is_small(m, 0);
    std::vector<R1csTerm> &terms = out.terms;
    terms.clear();
    terms.reserve(R.col.size());
    std::vector<uint64_t> sig(m, 0);
    std::vector<u32> wire2bool(R.n_wires, 0xFFFFFFFFu);
    for (size_t i = 0; i < bool_wire.size(); ++i)
        if (wire2bool[bool_wire[i]] == 0xFFFFFFFFu) wire2bool[bool_wire[i]] = (u32)i;
    std::vector<uint8_t> absorbed(bool_wire.size(), 0);
    const uint32_t qbits = F.qbits;
    uint64_t terms_general = 0;
    {
        size_t gi = 0;
        for (size_t row = 0; row < m; ++row) {
            const bool is_general = gi < general.size() && general[gi] == row;
            if (is_general) ++gi;
            uint64_t h = 1469598103934665603ull, cnt[3] = {0, 0, 0};
            bool small_shape = true;
            unsigned __int128 bound[3] = {0, 0, 0};   // of |sum| if every value met is below 2^16
            for (int blk = 0; blk < 3; ++blk) {
                row_ptr[3 * row + blk] = terms.size();
                if (!is_general) continue;
                uint64_t k = R.row_ptr[3 * row + blk];
                const uint64_t e = R.row_ptr[3 * row + blk + 1];
                while (k < e) {
                    const u32 loc = loc_of(R.col[k]);
                    const unsigned short kd = kind[R.coef[k]];
                    const int kk = kd & 0xFF;
                    // a run: plane bits at consecutive positions of one word, coefficients +-2^(s), +-2^(s+1), ...
                    if ((loc & OPERAND_BIT) && kk >= 1 && kk <= 4) {
                        const bool negc = kk == 2 || kk == 4;
                        const u32 s0 = kk <= 2 ? 0u : (u32)(kd >> 8), pos0 = loc & OPERAND_BITPOS_MASK;
                        uint64_t j = k + 1;
                        while (j < e) {
                            const u32 lj = loc_of(R.col[j]);
                            const unsigned short kj = kind[R.coef[j]];
                            const int kkj = kj & 0xFF;
                            if (!(lj & OPERAND_BIT) || kkj < 1 || kkj > 4 || (kkj == 2 || kkj == 4) != negc) break;
                            const u32 sj = kkj <= 2 ? 0u : (u32)(kj >> 8), pj = lj & OPERAND_BITPOS_MASK;
                            if (pj != pos0 + (u32)(j - k) || (pj >> 5) != (pos0 >> 5) || sj != s0 + (u32)(j - k)) break;
                            ++j;
                        }
                        const u32 n = (u32)(j - k);
                        if (s0 + n < qbits && s0 < 256) {  // the run's value is below 2^(s0 + n) <= 2^(qbits-1) < q
                            terms.push_back(R1csTerm{pos0 >> 5, 0u,
                                                     (negc ? 6u : 5u) | (s0 << 8) | ((pos0 & 31u) << 16) | ((n - 1u) << 21),
                                                     0xFFFFFFFFu});
                            if (s0 + n > R1CS_SMALL_MAX_BITS) small_shape = false;
                            else bound[blk] += (unsigned __int128)1 << (s0 + n);
                            h = (h ^ (negc ? 6u : 5u)) * 1099511628211ull;
                            ++cnt[blk];
                            k = j;
                            continue;
                        }
                    }
                    u32 brow = 0xFFFFFFFFu;
                    const u32 bi = wire2bool[R.col[k]];
                    if (bi != 0xFFFFFFFFu && !absorbed[bi]) {
                        absorbed[bi] = 1;
                        brow = bool_row[bi];
                    }
                    terms.push_back(R1csTerm{loc, R.coef[k], kd, brow});
                    // small by shape: +-1 / +-2^k with a small k, on a wire that is not a range-checked wide value (a wire the
                    // lowering bounds by more than 16 bits - a limb, a word - would fail the run-time test in every instance;
                    // a wire it knows nothing about is decided by the run)
                    const bool limb = T && T->wit_bits[R.col[k]] > 16 && T->wit_bits[R.col[k]] <= 128;   // (a bound near the field size is no bound)
                    if (kk < 1 || kk > 4 || (u32)(kd >> 8) > R1CS_SMALL_MAX_SHIFT || limb) small_shape = false;
                    else bound[blk] += (unsigned __int128)1 << (16 + (kk <= 2 ? 0u : (u32)(kd >> 8)));
                    h = (h ^ (u32)kk) * 1099511628211ull;
                    ++cnt[blk];
                    ++k;
                }
            }
            if (is_general) {
                const uint64_t total = std::min<uint64_t>(cnt[0] + cnt[1] + cnt[2], 0xFFFF);
                terms_general += cnt[0] + cnt[1] + cnt[2];
                sig[row] = (total << 48) | ((std::min<uint64_t>(cnt[0], 255)) << 40) | ((std::min<uint64_t>(cnt[1], 255)) << 32) | (h & 0xFFFFFFFFull);
                const unsigned __int128 lim = (unsigned __int128)1 << R1CS_SMALL_SUM_BITS;
                is_small[row] = want_small && small_shape && cnt[0] <= R1CS_SMALL_MAX_TERMS && cnt[1] <= R1CS_SMALL_MAX_TERMS &&
                                cnt[2] <= R1CS_SMALL_MAX_TERMS && bound[0] < lim && bound[1] < lim && bound[2] < lim;
            }
        }
        row_ptr[3 * m] = terms.size();
    }
    // rows sorted by structure so that neighbouring work items have equal length and branch alike
    std::stable_sort(general.begin(), general.end(), [&](u32 x, u32 y) { return sig[x] > sig[y]; });
    out.perm.clear();
    out.perm_small.clear();
    uint64_t terms_small = 0;
    for (u32 row : general) {
        if (is_small[row]) { out.perm_small.push_back(row); terms_small += sig[row] >> 48; }
        else out.perm.push_back(row);
    }
    // the integer-row pass pays when most rows take it (hash circuits: 98 %); a few rows small by shape among rows of limbs
    // (big-integer circuits: 2 %, and their unbounded wires are wide in every instance) stay with the general kernel
    if ((out.perm_small.size() < 1024 || out.perm_small.size() * 4 < general.size()) && !out.perm_small.empty() &&
        !getenv("CW_R1CS_SMALL_ALWAYS")) {
        out.perm = general;
        out.perm_small.clear();
        terms_small = 0;
    }
    {
        size_t o = 0;
        for (size_t i = 0; i < bool_wire.size(); ++i)
            if (!absorbed[i]) { bool_wire[o] = loc_of(bool_wire[i]); bool_row[o] = bool_row[i]; ++o; }
        bool_wire.resize(o);
        bool_row.resize(o);
    }
    // the integer rows' own term list (r1cs_small.h): groups of 32 rows, interleaved 8-byte records, uniform counts per group
    out.srecs.clear();
    out.sbrow.clear();
    out.sgroups.clear();
    {
        const size_t ns = out.perm_small.size();
        const u32 pad_loc = loc_of(0) & (SM_BIT | SM_BITPOS);   // the constant one: a value that is never wide; coefficient 0
        bool any_brow = false;
        for (size_t g0 = 0; g0 < ns; g0 += 32) {
            const size_t gn = std::min<size_t>(32, ns - g0);
            u32 n[3] = {0, 0, 0};
            for (size_t r = 0; r < gn; ++r)
                for (int blk = 0; blk < 3; ++blk)
                    n[blk] = std::max<u32>(n[blk], (u32)(row_ptr[3 * (size_t)out.perm_small[g0 + r] + blk + 1] -
                                                         row_ptr[3 * (size_t)out.perm_small[g0 + r] + blk]));
            const size_t base = out.srecs.size();
            if (base + (size_t)(n[0] + n[1] + n[2]) * 32 > 0xFFFFFFFFull) throw std::runtime_error("R1CS too large for the integer-row term list");
            out.sgroups.push_back((u32)base);
            out.sgroups.push_back(n[0] | (n[1] << 8) | (n[2] << 16));
            out.srecs.resize(base + (size_t)(n[0] + n[1] + n[2]) * 32, R1csSmallRec{pad_loc, SM_PAD});
            out.sbrow.resize(out.srecs.size(), 0xFFFFFFFFu);
            u32 t0 = 0;
            for (int blk = 0; blk < 3; ++blk) {
                for (size_t r = 0; r < gn; ++r) {
                    const u32 row = out.perm_small[g0 + r];
                    const unsigned long long b = row_ptr[3 * (size_t)row + blk], e = row_ptr[3 * (size_t)row + blk + 1];
                    for (unsigned long long k = b; k < e; ++k) {
                        const R1csTerm &tm = terms[k];
                        const u32 kd = tm.kind & 0xFFu, sh = (tm.kind >> 8) & 0xFFu;
                        R1csSmallRec rec;
                        if (kd >= 5u) {
                            rec.loc = (tm.loc & SM_LOC) | SM_RUN | (kd == 6u ? SM_NEG : 0u);
                            rec.mag = ((tm.kind >> 16) & 31u) | (((tm.kind >> 21) & 31u) << 5) | (sh << 10);
                        } else {
                            rec.loc = (tm.loc & (SM_BIT | SM_BITPOS)) | ((kd == 2u || kd == 4u) ? SM_NEG : 0u);   // (slot ids have 24 bits)
                            rec.mag = kd <= 2u ? 0u : sh;
                            if (tm.brow != 0xFFFFFFFFu) {
                                if (tm.loc & OPERAND_BIT) throw std::runtime_error("boolean row on a plane bit");
                                rec.loc |= SM_BROW;
                                any_brow = true;
                            }
                        }
                        const size_t at = base + ((size_t)t0 + (size_t)(k - b)) * 32 + r;
                        out.srecs[at] = rec;
                        out.sbrow[at] = tm.brow;
                    }
                }
                t0 += n[blk];
            }
        }
        if (!any_brow) out.sbrow.clear();
    }
    out.bool_loc = bool_wire;
    out.bool_row = bool_row;
    out.n_terms = terms.size();
    const size_t n_gen = out.perm.size();
    out.mean_row_terms = n_gen ? (u32)((terms_general - terms_small) / n_gen) : 0;
}

}  // namespace cw
