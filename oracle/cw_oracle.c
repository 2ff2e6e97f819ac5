/*
 * CPU ORACLE (TEST INFRASTRUCTURE — never linked into or called by the product).
 *
 * Plain-C restatement of the reference's witness-calculation path for a circuit description
 * (.cb2c, circom_b200/circuit.py):
 *
 *   field arithmetic   c_elements/generic/fr.cpp — Fr_rawAdd/Sub/Neg :19-86, CIOS Montgomery
 *                      product Fr_rawMMul :110-164 (4 x u64 limbs, np = -q^-1 mod 2^64),
 *                      comparisons on the signed view :1184-1218, bit operations with the
 *                      lboMask wrap :293-327,366-376, shifts :329-364,1995-2027,2157-2307,
 *                      Fr_inv / Fr_idiv / Fr_mod / Fr_pow :2835-2912 (GMP there, schoolbook here);
 *                      value-level semantics only: every witness value the reference writes goes
 *                      through Fr_toLongNormal (common/main.cpp:330);
 *   execution model    generated code + Circom_CalcWit: components created with
 *                      inputCounter = number_of_inputs (template.rs:204-209), a store into a
 *                      sub-component input decrements it and runs the sub-component at zero
 *                      (store_bucket.rs:660-734), input-less templates run at creation
 *                      (template.rs:274-278); signal 0 is the constant 1 (calcwit.cpp:34);
 *                      `===` asserts abort at the first failure (assert_bucket.rs:70-88);
 *   witness            witness[i] = signalValues[witness2SignalList[i]] (calcwit.hpp:54-56),
 *                      here the identity list (all signals), 32-byte canonical LE (main.cpp:328-332).
 *
 * Pinned against the compiled reference (oracle/_ref, the reference's own fr.cpp + runtime) by
 * tests/test_oracle_ref.py and tests/test_oracle_c.py.
 *
 * Build: gcc -O2 -shared -fPIC -o oracle/libcw_oracle.so oracle/cw_oracle.c
 */
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

typedef unsigned __int128 u128;
typedef uint64_t u64;
typedef uint32_t u32;

typedef struct { u64 v[4]; } fe;

typedef struct {
    fe q, half, r2;
    u64 np;
    u32 qbits;
} field_t;

/* ---- raw helpers ------------------------------------------------------------------------- */
static u64 add4(fe *r, const fe *a, const fe *b) {
    u128 c = 0;
    for (int i = 0; i < 4; ++i) { c += (u128)a->v[i] + b->v[i]; r->v[i] = (u64)c; c >>= 64; }
    return (u64)c;
}
static u64 sub4(fe *r, const fe *a, const fe *b) {
    u64 br = 0;
    for (int i = 0; i < 4; ++i) {
        u128 t = (u128)a->v[i] - b->v[i] - br;
        r->v[i] = (u64)t;
        br = (u64)(t >> 64) & 1;
    }
    return br;
}
static int cmp4(const fe *a, const fe *b) {
    for (int i = 3; i >= 0; --i) if (a->v[i] != b->v[i]) return a->v[i] < b->v[i] ? -1 : 1;
    return 0;
}
static int is_zero4(const fe *a) { return (a->v[0] | a->v[1] | a->v[2] | a->v[3]) == 0; }
static fe fe_u64(u64 x) { fe r = {{x, 0, 0, 0}}; return r; }

/* ---- field ------------------------------------------------------------------------------- */
static void f_add(const field_t *F, fe *r, const fe *a, const fe *b) {   /* Fr_rawAdd :19-27 */
    u64 c = add4(r, a, b);
    if (c || cmp4(r, &F->q) >= 0) sub4(r, r, &F->q);
}
static void f_sub(const field_t *F, fe *r, const fe *a, const fe *b) {   /* Fr_rawSub :39-47 */
    if (sub4(r, a, b)) add4(r, r, &F->q);
}
static void f_neg(const field_t *F, fe *r, const fe *a) {                /* Fr_rawNeg :76-86 */
    if (is_zero4(a)) *r = fe_u64(0); else sub4(r, &F->q, a);
}
static void f_mmul(const field_t *F, fe *r, const fe *a, const fe *b) {  /* Fr_rawMMul :110-164 */
    u64 t[6] = {0, 0, 0, 0, 0, 0};
    for (int i = 0; i < 4; ++i) {
        u128 c = 0;
        for (int j = 0; j < 4; ++j) { c += (u128)a->v[j] * b->v[i] + t[j]; t[j] = (u64)c; c >>= 64; }
        c += t[4]; t[4] = (u64)c; t[5] = (u64)(c >> 64);
        u64 m = t[0] * F->np;
        c = (u128)m * F->q.v[0] + t[0]; c >>= 64;
        for (int j = 1; j < 4; ++j) { c += (u128)m * F->q.v[j] + t[j]; t[j - 1] = (u64)c; c >>= 64; }
        c += t[4]; t[3] = (u64)c; t[4] = t[5] + (u64)(c >> 64);
    }
    fe x = {{t[0], t[1], t[2], t[3]}};
    if (t[4] || cmp4(&x, &F->q) >= 0) sub4(&x, &x, &F->q);
    *r = x;
}
static void f_mul(const field_t *F, fe *r, const fe *a, const fe *b) {   /* normal x normal */
    fe am;
    f_mmul(F, &am, a, &F->r2);   /* to Montgomery (Fr_toMontgomery :661) */
    f_mmul(F, r, &am, b);        /* Montgomery x normal -> normal (:449-465) */
}
static void f_pow(const field_t *F, fe *r, const fe *a, const fe *e) {   /* Fr_pow :2877-2893 */
    fe acc = fe_u64(1), base = *a;
    for (int i = 255; i >= 0; --i) {
        fe t;
        f_mul(F, &t, &acc, &acc); acc = t;
        if ((e->v[i >> 6] >> (i & 63)) & 1) { f_mul(F, &t, &acc, &base); acc = t; }
    }
    *r = acc;
}
static void f_inv(const field_t *F, fe *r, const fe *a) {                /* Fr_inv :2895-2906, inv(0)=0 */
    fe e, two = fe_u64(2);
    sub4(&e, &F->q, &two);
    f_pow(F, r, a, &e);
}
static int is_neg(const field_t *F, const fe *a) { return cmp4(a, &F->half) > 0; }
static int f_lt(const field_t *F, const fe *a, const fe *b) {            /* rltL1L2 :1208-1218 */
    int an = is_neg(F, a), bn = is_neg(F, b);
    if (an != bn) return an;
    return cmp4(a, b) < 0;
}
static void shl4(fe *r, const fe *a, unsigned k) {  /* (a << k) mod 2^256 */
    fe o = {{0, 0, 0, 0}};
    unsigned w = k / 64, s = k % 64;
    for (int i = 3; i >= (int)w; --i) {
        u64 x = a->v[i - w] << s;
        if (s && i - (int)w - 1 >= 0) x |= a->v[i - w - 1] >> (64 - s);
        o.v[i] = x;
    }
    *r = o;
}
static void shr4(fe *r, const fe *a, unsigned k) {
    fe o = {{0, 0, 0, 0}};
    unsigned w = k / 64, s = k % 64;
    for (unsigned i = 0; i + w < 4; ++i) {
        u64 x = a->v[i + w] >> s;
        if (s && i + w + 1 < 4) x |= a->v[i + w + 1] << (64 - s);
        o.v[i] = x;
    }
    *r = o;
}
static void wrap_bits(const field_t *F, fe *r) {                          /* lboMask + one conditional -q :293-303 */
    /* whole 64-bit words of the prime: 4 for the 256-bit primes, 1 for goldilocks (goldilocks/fr.hpp:177-181,255-270) */
    const unsigned top = (F->qbits - 1) / 64;
    u64 mask = F->qbits % 64 == 0 ? ~0ull : ((1ull << (F->qbits % 64)) - 1);
    r->v[top] &= mask;
    for (unsigned i = top + 1; i < 4; ++i) r->v[i] = 0;
    if (cmp4(r, &F->q) >= 0) sub4(r, r, &F->q);
}
static int shift_kind(const field_t *F, const fe *b, unsigned *k) {      /* :1995-2027,2157-2307 */
    if (!(b->v[1] | b->v[2] | b->v[3]) && b->v[0] < F->qbits) { *k = (unsigned)b->v[0]; return 0; }
    fe nb;
    sub4(&nb, &F->q, b);
    if (!(nb.v[1] | nb.v[2] | nb.v[3]) && nb.v[0] < F->qbits) { *k = (unsigned)nb.v[0]; return 1; }
    return 2;
}
static void f_shl(const field_t *F, fe *r, const fe *a, const fe *b) {
    unsigned k; int kind = shift_kind(F, b, &k);
    if (kind == 0) { shl4(r, a, k); wrap_bits(F, r); }
    else if (kind == 1) shr4(r, a, k);
    else *r = fe_u64(0);
}
static void f_shr(const field_t *F, fe *r, const fe *a, const fe *b) {
    unsigned k; int kind = shift_kind(F, b, &k);
    if (kind == 0) shr4(r, a, k);
    else if (kind == 1) { shl4(r, a, k); wrap_bits(F, r); }
    else *r = fe_u64(0);
}
/* floor division of canonical integers (mpz_fdiv_q / mpz_fdiv_r :2835-2875); returns 0 if b == 0 */
static int divmod4(fe *quo, fe *rem, const fe *a, const fe *b) {
    if (is_zero4(b)) return 0;
    fe q = {{0, 0, 0, 0}}, r = {{0, 0, 0, 0}};
    for (int i = 255; i >= 0; --i) {
        u64 top = r.v[3] >> 63;
        shl4(&r, &r, 1);
        r.v[0] |= (a->v[i >> 6] >> (i & 63)) & 1;
        if (top || cmp4(&r, b) >= 0) { sub4(&r, &r, b); q.v[i >> 6] |= 1ull << (i & 63); }
    }
    *quo = q; *rem = r;
    return 1;
}

enum { OP_NOP = 0, OP_MUL = 1, OP_DIV = 2, OP_ADD = 3, OP_SUB = 4, OP_POW = 5, OP_IDIV = 6, OP_MOD = 7,
       OP_SHL = 8, OP_SHR = 9, OP_LEQ = 10, OP_GEQ = 11, OP_LT = 12, OP_GT = 13, OP_EQ = 14, OP_NEQ = 15,
       OP_LOR = 16, OP_LAND = 17, OP_LNOT = 18, OP_BOR = 19, OP_BAND = 20, OP_BXOR = 21, OP_BNOT = 22,
       OP_NEG = 23, OP_COPY = 24, OP_SELECT = 25, OP_ASSERT = 26, OP_ASSERT_EQ = 27 };

/* one operator on canonical values; returns 0 on division by zero */
static int f_apply(const field_t *F, u32 op, fe *r, const fe *a, const fe *b, const fe *c) {
    fe t;
    switch (op) {
        case OP_MUL: f_mul(F, r, a, b); break;
        case OP_DIV: f_inv(F, &t, b); f_mul(F, r, a, &t); break;
        case OP_ADD: f_add(F, r, a, b); break;
        case OP_SUB: f_sub(F, r, a, b); break;
        case OP_POW: f_pow(F, r, a, b); break;
        case OP_IDIV: if (!divmod4(r, &t, a, b)) return 0; break;
        case OP_MOD: if (!divmod4(&t, r, a, b)) return 0; break;
        case OP_SHL: f_shl(F, r, a, b); break;
        case OP_SHR: f_shr(F, r, a, b); break;
        case OP_LT: *r = fe_u64(f_lt(F, a, b)); break;
        case OP_GT: *r = fe_u64(f_lt(F, b, a)); break;
        case OP_LEQ: *r = fe_u64(!f_lt(F, b, a)); break;
        case OP_GEQ: *r = fe_u64(!f_lt(F, a, b)); break;
        case OP_EQ: *r = fe_u64(cmp4(a, b) == 0); break;
        case OP_NEQ: *r = fe_u64(cmp4(a, b) != 0); break;
        case OP_LOR: *r = fe_u64(!is_zero4(a) || !is_zero4(b)); break;
        case OP_LAND: *r = fe_u64(!is_zero4(a) && !is_zero4(b)); break;
        case OP_LNOT: *r = fe_u64(is_zero4(a)); break;
        case OP_BOR: for (int i = 0; i < 4; ++i) r->v[i] = a->v[i] | b->v[i]; wrap_bits(F, r); break;
        case OP_BAND: for (int i = 0; i < 4; ++i) r->v[i] = a->v[i] & b->v[i]; wrap_bits(F, r); break;
        case OP_BXOR: for (int i = 0; i < 4; ++i) r->v[i] = a->v[i] ^ b->v[i]; wrap_bits(F, r); break;
        case OP_BNOT: for (int i = 0; i < 4; ++i) r->v[i] = ~a->v[i]; wrap_bits(F, r); break;
        case OP_NEG: f_neg(F, r, a); break;
        case OP_COPY: *r = *a; break;
        case OP_SELECT: *r = is_zero4(c) ? *b : *a; break;   /* Fr_isTrue(c) ? a : b */
        default: *r = fe_u64(0); break;
    }
    return 1;
}

/* ---- circuit description ------------------------------------------------------------------ */
enum { K_NONE = 0, K_OWN = 1, K_SUB = 2, K_CONST = 3, K_TMP = 4, K_ONE = 5 };
typedef struct { u32 op; u64 d, a, b, c; } irop;
typedef struct { u64 ref; u32 cid; } term;
typedef struct {
    u32 n_out, n_in, n_inter, n_own, n_sub, n_tmp, n_ops, n_cons, n_terms;
    u32 *subs; irop *ops; u32 *lc_len; term *terms;
    u64 total_signals;
} tmpl;
/* function bodies (FunctionCodeInfo, compiler/src/circuit_design/function.rs:91-126): register code with
 * jumps; called through CallBucket (call_bucket.rs:466-533) */
typedef struct { u32 n_params, n_regs, n_instr; irop *code; } func;
typedef struct {
    field_t F;
    u32 prime, n_consts, n_tm, main_tid, n_funcs;
    fe *consts;
    tmpl *tm;
    func *fn;
} circuit;

#define RK(r) ((int)((r) >> 56))
#define RSUB(r) ((u32)(((r) >> 32) & 0xFFFFFF))
#define RIDX(r) ((u32)(r))

static void field_init(field_t *F, u32 prime) {
    /* program_structure/src/utils/constants.rs:3-13: bn128, bls12381, grumpkin, pallas, vesta, secq256r1, bls12377, goldilocks */
    static const u64 Q[8][4] = {
        {0x43e1f593f0000001ULL, 0x2833e84879b97091ULL, 0xb85045b68181585dULL, 0x30644e72e131a029ULL},
        {0xffffffff00000001ULL, 0x53bda402fffe5bfeULL, 0x3339d80809a1d805ULL, 0x73eda753299d7d48ULL},
        {0x3c208c16d87cfd47ULL, 0x97816a916871ca8dULL, 0xb85045b68181585dULL, 0x30644e72e131a029ULL},
        {0x992d30ed00000001ULL, 0x224698fc094cf91bULL, 0x0000000000000000ULL, 0x4000000000000000ULL},
        {0x8c46eb2100000001ULL, 0x224698fc0994a8ddULL, 0x0000000000000000ULL, 0x4000000000000000ULL},
        {0xffffffffffffffffULL, 0x00000000ffffffffULL, 0x0000000000000000ULL, 0xffffffff00000001ULL},
        {0x0a11800000000001ULL, 0x59aa76fed0000001ULL, 0x60b44d1e5c37b001ULL, 0x12ab655e9a2ca556ULL},
        {0xffffffff00000001ULL, 0, 0, 0},
    };
    memcpy(F->q.v, Q[prime < 8 ? prime : 0], 32);
    for (int i = 0; i < 4; ++i) F->half.v[i] = (F->q.v[i] >> 1) | (i < 3 ? F->q.v[i + 1] << 63 : 0);
    u64 inv = 1;
    for (int i = 0; i < 6; ++i) inv *= 2 - F->q.v[0] * inv;
    F->np = (u64)0 - inv;
    F->qbits = 0;
    for (int i = 255; i >= 0; --i) if ((F->q.v[i >> 6] >> (i & 63)) & 1) { F->qbits = (u32)i + 1; break; }
    fe x = fe_u64(1);
    for (int i = 0; i < 512; ++i) f_add(F, &x, &x, &x);
    F->r2 = x;
}

typedef struct { const uint8_t *p, *end; int bad; } rd_t;
static u32 rd32(rd_t *r) { u32 v = 0; if (r->p + 4 > r->end) { r->bad = 1; return 0; } memcpy(&v, r->p, 4); r->p += 4; return v; }
static u64 rd64(rd_t *r) { u64 v = 0; if (r->p + 8 > r->end) { r->bad = 1; return 0; } memcpy(&v, r->p, 8); r->p += 8; return v; }

circuit *orc_load(const uint8_t *data, size_t len) {
    rd_t r = {data, data + len, 0};
    if (len < 32 || memcmp(data, "CB2C", 4)) return NULL;
    r.p += 4;
    if (rd32(&r) != 1) return NULL;
    circuit *c = (circuit *)calloc(1, sizeof(circuit));
    c->prime = rd32(&r); c->n_consts = rd32(&r); c->n_tm = rd32(&r); c->main_tid = rd32(&r);
    u32 n_names = rd32(&r);
    c->n_funcs = rd32(&r);
    field_init(&c->F, c->prime);
    c->consts = (fe *)calloc(c->n_consts ? c->n_consts : 1, sizeof(fe));
    for (u32 i = 0; i < c->n_consts; ++i) { if (r.p + 32 > r.end) { r.bad = 1; break; } memcpy(c->consts[i].v, r.p, 32); r.p += 32; }
    c->tm = (tmpl *)calloc(c->n_tm, sizeof(tmpl));
    for (u32 i = 0; i < c->n_tm && !r.bad; ++i) {
        tmpl *t = &c->tm[i];
        u32 nl = rd32(&r);
        r.p += (nl + 3) & ~3u;
        t->n_out = rd32(&r); t->n_in = rd32(&r); t->n_inter = rd32(&r); t->n_sub = rd32(&r);
        t->n_tmp = rd32(&r); t->n_ops = rd32(&r); t->n_cons = rd32(&r); t->n_terms = rd32(&r);
        t->n_own = t->n_out + t->n_in + t->n_inter;
        t->subs = (u32 *)calloc(t->n_sub ? t->n_sub : 1, 4);
        t->total_signals = t->n_own;
        for (u32 k = 0; k < t->n_sub; ++k) { t->subs[k] = rd32(&r); if (t->subs[k] < i) t->total_signals += c->tm[t->subs[k]].total_signals; else r.bad = 1; }
        t->ops = (irop *)calloc(t->n_ops ? t->n_ops : 1, sizeof(irop));
        for (u32 k = 0; k < t->n_ops; ++k) { t->ops[k].op = (u32)rd64(&r); t->ops[k].d = rd64(&r); t->ops[k].a = rd64(&r); t->ops[k].b = rd64(&r); t->ops[k].c = rd64(&r); }
        t->lc_len = (u32 *)calloc(t->n_cons * 3 + 1, 4);
        t->terms = (term *)calloc(t->n_terms ? t->n_terms : 1, sizeof(term));
        u32 ti = 0;
        for (u32 k = 0; k < t->n_cons * 3; ++k) {
            u32 n = (u32)rd64(&r);
            t->lc_len[k] = n;
            for (u32 j = 0; j < n && ti < t->n_terms; ++j, ++ti) { t->terms[ti].ref = rd64(&r); t->terms[ti].cid = (u32)rd64(&r); }
        }
    }
    for (u32 i = 0; i < n_names && !r.bad; ++i) { u32 nl = rd32(&r); r.p += ((nl + 3) & ~3u) + 8; }
    c->fn = (func *)calloc(c->n_funcs ? c->n_funcs : 1, sizeof(func));
    for (u32 i = 0; i < c->n_funcs && !r.bad; ++i) {
        func *f = &c->fn[i];
        u32 nl = rd32(&r);
        r.p += (nl + 3) & ~3u;
        f->n_params = rd32(&r); f->n_regs = rd32(&r); f->n_instr = rd32(&r);
        f->code = (irop *)calloc(f->n_instr ? f->n_instr : 1, sizeof(irop));
        for (u32 k = 0; k < f->n_instr; ++k) { f->code[k].op = (u32)rd64(&r); f->code[k].d = rd64(&r); f->code[k].a = rd64(&r); f->code[k].b = rd64(&r); f->code[k].c = rd64(&r); }
    }
    if (r.bad || r.p > r.end) return NULL;
    return c;
}

u64 orc_total_signals(const circuit *c) { return 1 + c->tm[c->main_tid].total_signals; }
u32 orc_n_inputs(const circuit *c) { return c->tm[c->main_tid].n_in; }

/* ---- execution ---------------------------------------------------------------------------- */
typedef struct { u32 tid; u64 start; u32 counter; int ran; } comp;
typedef struct {
    const circuit *c;
    fe *sig;
    unsigned char *set;
    int32_t status;     /* 0 ok; k+1 first failed assert; -1 division by zero; -2 malformed program */
    u32 n_asserts;
    int stop_on_assert;
} ctx_t;

/* one function call: variables are registers, loops / branches test Fr_isTrue (loop_bucket.rs:76-91,
 * branch_bucket.rs:100-122), array variables are indexed through Fr_toInt (compute_bucket.rs:361-363).
 * returns 0 ok, -1 division by zero, -2 bad index / runaway */
#define MAX_RESULTS 64
/* result[0 .. *n_res): RET with a count in operand b returns that many consecutive registers (return_bucket.rs with_size) */
static int run_func(const circuit *c, const func *f, const fe *args, fe *result, u32 *n_res) {
    fe *regs = (fe *)calloc(f->n_regs ? f->n_regs : 1, sizeof(fe));
    for (u32 i = 0; i < f->n_params; ++i) regs[i] = args[i];
    fe zero = fe_u64(0);
    u32 pc = 0;
    int rc = -2;
    for (long step = 0; step < (1L << 22) && pc < f->n_instr; ++step) {
        const irop *o = &f->code[pc++];
        const fe *arg[3] = {&zero, &zero, &zero};
        u64 refs[3] = {o->a, o->b, o->c};
        for (int j = 0; j < 3; ++j) {
            if (RK(refs[j]) == K_TMP) arg[j] = &regs[RIDX(refs[j])];
            else if (RK(refs[j]) == K_CONST) arg[j] = &c->consts[RIDX(refs[j])];
        }
        if (o->op == 40) { pc = RIDX(o->a); continue; }                          /* JMP */
        if (o->op == 41) { if (is_zero4(arg[0])) pc = RIDX(o->b); continue; }      /* JZ */
        if (o->op == 42) {                                                         /* RET */
            u32 cnt = RK(o->b) == 0 ? RIDX(o->b) : 0;
            if (cnt > 1) {
                if (RK(o->a) != K_TMP || RIDX(o->a) + cnt > f->n_regs || cnt > MAX_RESULTS) break;
                for (u32 k = 0; k < cnt; ++k) result[k] = regs[RIDX(o->a) + k];
                *n_res = cnt;
            } else { result[0] = *arg[0]; *n_res = 1; }
            rc = 0;
            break;
        }
        if (o->op == 45) {                                                         /* nested CALL of an earlier function */
            u32 fid = RIDX(o->a), want = RK(o->c) == 0 && RIDX(o->c) > 1 ? RIDX(o->c) : 1, got = 0;
            if (fid >= c->n_funcs || &c->fn[fid] >= f) break;
            const func *g = &c->fn[fid];
            if (RIDX(o->b) + g->n_params > f->n_regs || RIDX(o->d) + want > f->n_regs) break;
            fe res[MAX_RESULTS];
            int rc2 = run_func(c, g, &regs[RIDX(o->b)], res, &got);
            if (rc2) { rc = rc2; break; }
            if (got < want) break;
            for (u32 k = 0; k < want; ++k) regs[RIDX(o->d) + k] = res[k];
            continue;
        }
        if (o->op == 43 || o->op == 44) {                                          /* LOADX / STOREX */
            const fe *ix = arg[1];
            /* the extent of the array, when the producer wrote it (LOADX: operand c, STOREX: operand d; docs/CB2C.md) */
            const u64 ext = o->op == 43 ? (RK(o->c) == 0 ? RIDX(o->c) : 0) : (RK(o->d) == 0 ? RIDX(o->d) : 0);
            const u64 lim = ext && RIDX(o->a) + ext <= f->n_regs ? RIDX(o->a) + ext : f->n_regs;
            if (ix->v[1] | ix->v[2] | ix->v[3] || ix->v[0] + RIDX(o->a) >= lim) break;
            u32 i = (u32)ix->v[0] + RIDX(o->a);
            if (o->op == 43) regs[RIDX(o->d)] = regs[i]; else regs[i] = *arg[2];
            continue;
        }
        fe v;
        if (!f_apply(&c->F, o->op, &v, arg[0], arg[1], arg[2])) { rc = -1; break; }
        regs[RIDX(o->d)] = v;
    }
    free(regs);
    return rc;
}

static void run_comp(ctx_t *x, comp *me) {
    const circuit *c = x->c;
    const tmpl *t = &c->tm[me->tid];
    me->ran = 1;
    fe *tmp = (fe *)malloc(sizeof(fe) * (t->n_tmp ? t->n_tmp : 1));
    comp *subs = (comp *)calloc(t->n_sub ? t->n_sub : 1, sizeof(comp));
    u64 off = me->start + t->n_own;
    for (u32 i = 0; i < t->n_sub; ++i) {                       /* CreateCmp buckets */
        const tmpl *st = &c->tm[t->subs[i]];
        subs[i].tid = t->subs[i]; subs[i].start = off; subs[i].counter = st->n_in; subs[i].ran = 0;
        off += st->total_signals;
        if (st->n_in == 0) run_comp(x, &subs[i]);
    }
    fe zero = fe_u64(0), one = fe_u64(1);
    fe argstack[64];
    u32 n_args = 0;
    for (u32 k = 0; k < t->n_ops && x->status != -1 && x->status != -2; ++k) {
        const irop *o = &t->ops[k];
        if (o->op == 29) continue;   /* LOG: prints, computes nothing (log_bucket.rs:104-162) */
        const fe *arg[3] = {&zero, &zero, &zero};
        u64 refs[3] = {o->a, o->b, o->c};
        for (int j = 0; j < 3; ++j) {
            u64 r = refs[j];
            switch (RK(r)) {
                case K_OWN: arg[j] = &x->sig[me->start + RIDX(r)]; if (!x->set[me->start + RIDX(r)]) x->status = -2; break;
                case K_SUB: { u64 g = subs[RSUB(r)].start + RIDX(r); arg[j] = &x->sig[g]; if (!x->set[g]) x->status = -2; break; }
                case K_CONST: arg[j] = &c->consts[RIDX(r)]; break;
                case K_TMP: arg[j] = &tmp[RIDX(r)]; break;
                case K_ONE: arg[j] = &one; break;
                default: break;
            }
        }
        if (x->status == -2) break;
        if (o->op == 46) { if (n_args < 64) argstack[n_args++] = *arg[0]; continue; }     /* ARG */
        if (o->op == 45) {                                                              /* CALL */
            u32 fid = RIDX(o->a), n = RIDX(o->b);
            fe res[MAX_RESULTS];
            u32 got = 0, want = RK(o->c) == 0 && RIDX(o->c) > 1 ? RIDX(o->c) : 1;
            if (fid >= c->n_funcs || n > n_args) { x->status = -2; break; }
            int rc = run_func(c, &c->fn[fid], &argstack[n_args - n], res, &got);
            n_args -= n;
            if (rc) { x->status = rc; break; }
            if (got < want || RIDX(o->d) + want > t->n_tmp) { x->status = -2; break; }
            for (u32 k = 0; k < want; ++k) tmp[RIDX(o->d) + k] = res[k];   /* n results in consecutive temporaries */
            continue;
        }
        if (o->op == OP_ASSERT_EQ || o->op == OP_ASSERT) {
            u32 id = x->n_asserts++;
            int ok = o->op == OP_ASSERT_EQ ? cmp4(arg[0], arg[1]) == 0 : !is_zero4(arg[0]);
            if (!ok && x->status == 0) { x->status = (int32_t)id + 1; if (x->stop_on_assert) break; }
            continue;
        }
        fe v;
        if (!f_apply(&c->F, o->op, &v, arg[0], arg[1], arg[2])) { x->status = -1; break; }
        switch (RK(o->d)) {
            case K_TMP: tmp[RIDX(o->d)] = v; break;
            case K_OWN: { u64 g = me->start + RIDX(o->d); if (x->set[g]) x->status = -2; x->sig[g] = v; x->set[g] = 1; break; }
            case K_SUB: {
                comp *sc = &subs[RSUB(o->d)];
                const tmpl *st = &c->tm[sc->tid];
                u64 g = sc->start + RIDX(o->d);
                if (x->set[g]) x->status = -2;
                x->sig[g] = v; x->set[g] = 1;
                u32 li = RIDX(o->d);
                if (li >= st->n_out && li < st->n_out + st->n_in) {   /* store_bucket.rs:660-734 */
                    if (--sc->counter == 0) run_comp(x, sc);
                }
                break;
            }
            default: x->status = -2; break;
        }
    }
    free(subs);
    free(tmp);
}

/* inputs[n_in][4] canonical, witness[total_signals][4]; returns status (see ctx_t) */
int32_t orc_run(const circuit *c, const u64 *inputs, u64 *witness) {
    const tmpl *M = &c->tm[c->main_tid];
    u64 S = orc_total_signals(c);
    ctx_t x;
    x.c = c; x.status = 0; x.n_asserts = 0; x.stop_on_assert = 0;
    x.sig = (fe *)witness;
    x.set = (unsigned char *)calloc(S, 1);
    memset(witness, 0, S * 32);
    x.sig[0] = fe_u64(1); x.set[0] = 1;
    for (u32 i = 0; i < M->n_in; ++i) { memcpy(x.sig[1 + M->n_out + i].v, inputs + 4 * (u64)i, 32); x.set[1 + M->n_out + i] = 1; }
    comp mc = {c->main_tid, 1, 0, 0};
    run_comp(&x, &mc);
    if (x.status == 0) for (u64 i = 0; i < S; ++i) if (!x.set[i]) { x.status = -2; break; }
    free(x.set);
    return x.status;
}

/* ---- R1CS check: rows in component pre-order (parent's constraints, then its sub-components) - */
static void r1cs_walk(const circuit *c, u32 tid, u64 start, const fe *w, int64_t *row, int64_t *first_bad) {
    const tmpl *t = &c->tm[tid];
    u64 *offs = (u64 *)malloc(8 * (t->n_sub ? t->n_sub : 1));
    u64 off = start + t->n_own;
    for (u32 i = 0; i < t->n_sub; ++i) { offs[i] = off; off += c->tm[t->subs[i]].total_signals; }
    u32 ti = 0;
    for (u32 k = 0; k < t->n_cons; ++k) {
        fe acc[3];
        for (int m = 0; m < 3; ++m) {
            acc[m] = fe_u64(0);
            for (u32 j = 0; j < t->lc_len[3 * k + m]; ++j, ++ti) {
                u64 r = t->terms[ti].ref, g = 0;
                if (RK(r) == K_OWN) g = start + RIDX(r); else if (RK(r) == K_SUB) g = offs[RSUB(r)] + RIDX(r);
                fe p;
                f_mul(&c->F, &p, &c->consts[t->terms[ti].cid], &w[g]);
                f_add(&c->F, &acc[m], &acc[m], &p);
            }
        }
        fe ab;
        f_mul(&c->F, &ab, &acc[0], &acc[1]);
        if (cmp4(&ab, &acc[2]) != 0 && *first_bad < 0) *first_bad = *row;
        ++*row;
    }
    for (u32 i = 0; i < t->n_sub; ++i) r1cs_walk(c, t->subs[i], offs[i], w, row, first_bad);
    free(offs);
}
int64_t orc_r1cs_check(const circuit *c, const u64 *witness) {
    int64_t row = 0, first_bad = -1;
    r1cs_walk(c, c->main_tid, 1, (const fe *)witness, &row, &first_bad);
    return first_bad;
}

/* single operator, canonical in/out (for pinning against the reference library); 0 on div by zero */
int orc_apply(u32 prime, u32 op, const u64 *a, const u64 *b, const u64 *c3, u64 *r) {
    static field_t F[8]; static int init[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    if (prime >= 8) return -1;
    if (!init[prime]) { field_init(&F[prime], prime); init[prime] = 1; }
    fe z = fe_u64(0);
    return f_apply(&F[prime], op, (fe *)r, (const fe *)a, b ? (const fe *)b : &z, c3 ? (const fe *)c3 : &z);
}

/* ---- throughput runner for the CPU baseline: `threads` workers, each reusing one witness buffer
 * (the reference allocates signalValues once per process, calcwit.cpp:33); returns the number of
 * instances whose status was 0.  inputs[n][n_in][4]. */
#include <pthread.h>
typedef struct { const circuit *c; const u64 *inputs; long n; volatile long *next; long ok; } many_t;
static void *many_worker(void *p) {
    many_t *m = (many_t *)p;
    u64 S = orc_total_signals(m->c);
    u32 n_in = orc_n_inputs(m->c);
    u64 *wit = (u64 *)malloc(S * 32);
    for (;;) {
        long i = __sync_fetch_and_add(m->next, 1);
        if (i >= m->n) break;
        if (orc_run(m->c, m->inputs + (u64)i * n_in * 4, wit) == 0) m->ok++;
    }
    free(wit);
    return NULL;
}
long orc_run_many(const circuit *c, const u64 *inputs, long n, int threads) {
    if (threads < 1) threads = 1;
    pthread_t *th = (pthread_t *)malloc(sizeof(pthread_t) * threads);
    many_t *ms = (many_t *)calloc(threads, sizeof(many_t));
    volatile long next = 0;
    for (int t = 0; t < threads; ++t) {
        ms[t].c = c; ms[t].inputs = inputs; ms[t].n = n; ms[t].next = &next; ms[t].ok = 0;
        pthread_create(&th[t], NULL, many_worker, &ms[t]);
    }
    long ok = 0;
    for (int t = 0; t < threads; ++t) { pthread_join(th[t], NULL); ok += ms[t].ok; }
    free(th); free(ms);
    return ok;
}

/* ---- polynomial evaluation, for spot checks of transforms too large for a Python sum: out = sum_{i<n} coef[i] x^i
 * (coef[n][4] and x canonical, below q).  Horner's rule over `threads` contiguous slices of the coefficients; slice t
 * starting at lo contributes x^lo times its own Horner value.  Returns 0 for an unknown prime. */
typedef struct { const field_t *F; const fe *coef; u64 lo, hi; fe xm, acc; } horner_t;
static void *horner_worker(void *p) {
    horner_t *h = (horner_t *)p;
    fe acc = fe_u64(0), t;
    for (u64 i = h->hi; i-- > h->lo;) {
        f_mmul(h->F, &t, &acc, &h->xm);   /* acc * x: the Montgomery image of x times a normal value is normal */
        f_add(h->F, &acc, &t, &h->coef[i]);
    }
    h->acc = acc;
    return NULL;
}
int orc_poly_eval(u32 prime, const u64 *coef, u64 n, const u64 *x, int threads, u64 *out) {
    if (prime >= 8) return 0;
    field_t F;
    field_init(&F, prime);
    if (threads < 1) threads = 1;
    if ((u64)threads > n) threads = n ? (int)n : 1;
    pthread_t *th = (pthread_t *)malloc(sizeof(pthread_t) * threads);
    horner_t *hs = (horner_t *)calloc(threads, sizeof(horner_t));
    fe xm;
    f_mmul(&F, &xm, (const fe *)x, &F.r2);
    for (int t = 0; t < threads; ++t) {
        hs[t].F = &F; hs[t].coef = (const fe *)coef; hs[t].xm = xm;
        hs[t].lo = n * t / threads; hs[t].hi = n * (t + 1) / threads;
        pthread_create(&th[t], NULL, horner_worker, &hs[t]);
    }
    fe sum = fe_u64(0);
    for (int t = 0; t < threads; ++t) {
        pthread_join(th[t], NULL);
        fe e = fe_u64(hs[t].lo), xl, p;
        f_pow(&F, &xl, (const fe *)x, &e);
        f_mul(&F, &p, &hs[t].acc, &xl);
        f_add(&F, &sum, &sum, &p);
    }
    memcpy(out, sum.v, 32);
    free(th); free(hs);
    return 1;
}

void orc_free(circuit *c) {
    if (!c) return;
    for (u32 i = 0; i < c->n_tm; ++i) { free(c->tm[i].subs); free(c->tm[i].ops); free(c->tm[i].lc_len); free(c->tm[i].terms); }
    for (u32 i = 0; i < c->n_funcs; ++i) free(c->fn[i].code);
    free(c->fn); free(c->tm); free(c->consts); free(c);
}
