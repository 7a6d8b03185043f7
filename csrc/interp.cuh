// interp.cuh — the expression interpreter shared by the generic aggregate kernel (agg.cu) and the
// sort / filter kernels (sort.cu): postfix bytecode lowered by plan.cpp, warp-uniform dispatch.
#pragma once
#include "dev_common.cuh"
#include "in_set.h"

namespace bk {

// ------------------------------------------------------------------------------------------
// generic path: the lowered expression program is interpreted per row (any predicate, computed
// keys and arguments, multi-column keys).  Postfix bytecode, warp-uniform dispatch.
// ------------------------------------------------------------------------------------------
// OP_DATEFN's calendar code (datetime.h), out of line: one call site keeps it out of run_program's registers
static __device__ __noinline__ uint64_t date_fn(uint32_t fn, uint32_t arg, uint64_t x, uint64_t x2) { return dt_date_fn((int)fn, (int)arg, x, x2); }
// OP_IN_SET's probe of the hashed set at device address `set` (in_set.h), out of line for the same reason
static __device__ __noinline__ bool in_set_probe(uint64_t set, uint64_t x, uint32_t vclass) { return in_set_contains((const uint64_t*)set, x, (int)vclass); }

// `brow`: row of the join's build side; LOAD_COL instructions with c == 1 read there (the joined row of
// Joiner::construct_result_batch, src/exec/joiner.cpp:633-685, without materialising it)
static __device__ __noinline__ void run_program(const Program& p, const DevCol* cols, int64_t row, uint64_t* out, uint32_t& out_null, int64_t brow = -1) {
    uint64_t st[STACK_DEPTH];
    uint32_t nul = 0;  // bit d set = stack entry d is NULL
    int sp = 0;
    out_null = 0;
#pragma unroll 1
    for (int pc = 0; pc < p.n_instr; pc++) {
        const Instr in = p.code[pc];
        switch (in.op) {
            case OP_LOAD_COL: {
                const DevCol& c = cols[in.a];
                const int64_t r = in.c ? brow : row;
                if (r < 0) { st[sp] = 0; nul |= 1u << sp; sp++; break; }   // the NULL-extended side of an outer join's unmatched row (Joiner::construct_null_result_batch)
                st[sp] = in.b == 4 ? (uint64_t)r : in.b == 3 ? (uint64_t)__ldg((const uint32_t*)c.values + r)
                       : in.b ? __ldg((const unsigned long long*)c.values + 2 * r + (in.b - 1)) : load_elem(c, r);
                nul = elem_is_null(c, r) ? (nul | (1u << sp)) : (nul & ~(1u << sp));
                sp++;
            } break;
            case OP_CONST:
                st[sp] = p.cbits[in.a];
                nul = ((p.cnull >> in.a) & 1ull) ? (nul | (1u << sp)) : (nul & ~(1u << sp));
                sp++;
                break;
            case OP_CAST:
                if (!((nul >> (sp - 1)) & 1u)) st[sp - 1] = cast_prim(st[sp - 1], in.a, in.b);
                break;
            case OP_CMP: {
                sp--;
                const bool n = ((nul >> sp) | (nul >> (sp - 1))) & 1u;
                st[sp - 1] = n ? 0 : (cmp_vals(in.a, in.b, st[sp - 1], st[sp]) ? 1ull : 0ull);
                nul = n ? (nul | (1u << (sp - 1))) : (nul & ~(1u << (sp - 1)));
            } break;
            case OP_ARITH: {
                sp--;
                const bool n = ((nul >> sp) | (nul >> (sp - 1))) & 1u;
                uint64_t x = st[sp - 1], y = st[sp], r;
                if (in.b == VC_F64) {
                    double dx = bits_f64(x), dy = bits_f64(y);
                    r = f64_bits(in.a == BK_FT_ADD ? __dadd_rn(dx, dy) : (in.a == BK_FT_MINUS ? __dsub_rn(dx, dy) : __dmul_rn(dx, dy)));
                } else r = in.a == BK_FT_ADD ? x + y : (in.a == BK_FT_MINUS ? x - y : x * y);
                st[sp - 1] = r;
                nul = n ? (nul | (1u << (sp - 1))) : (nul & ~(1u << (sp - 1)));
            } break;
            case OP_DIV_F64: {
                sp--;
                bool n = ((nul >> sp) | (nul >> (sp - 1))) & 1u;
                const double dy = bits_f64(st[sp]);
                if (!n && dy == 0.0) n = true;  // NULL on zero divisor
                if (!n) st[sp - 1] = f64_bits(__ddiv_rn(bits_f64(st[sp - 1]), dy));
                nul = n ? (nul | (1u << (sp - 1))) : (nul & ~(1u << (sp - 1)));
            } break;
            case OP_MOD: {
                sp--;
                bool n = ((nul >> sp) | (nul >> (sp - 1))) & 1u;
                if (!n && st[sp] == 0) n = true;
                if (!n) {
                    if (in.b == VC_U64) st[sp - 1] = st[sp - 1] % st[sp];
                    else { int64_t y = (int64_t)st[sp]; st[sp - 1] = y == -1 ? 0 : (uint64_t)((int64_t)st[sp - 1] % y); }
                }
                nul = n ? (nul | (1u << (sp - 1))) : (nul & ~(1u << (sp - 1)));
            } break;
            case OP_BIT: {
                sp--;
                const bool n = ((nul >> sp) | (nul >> (sp - 1))) & 1u;
                uint64_t x = st[sp - 1], y = st[sp], r;
                switch (in.a) {
                    case BK_FT_BIT_AND: r = x & y; break;
                    case BK_FT_BIT_OR: r = x | y; break;
                    case BK_FT_BIT_XOR: r = x ^ y; break;
                    case BK_FT_LS: r = y >= 64 ? 0 : x << y; break;
                    default: r = y >= 64 ? 0 : x >> y; break;
                }
                st[sp - 1] = r;
                nul = n ? (nul | (1u << (sp - 1))) : (nul & ~(1u << (sp - 1)));
            } break;
            case OP_BIT_NOT: st[sp - 1] = ~st[sp - 1]; break;
            case OP_NEG:
                st[sp - 1] = in.b == VC_F64 ? f64_bits(-bits_f64(st[sp - 1])) : (uint64_t)0 - st[sp - 1];
                break;
            case OP_LOGIC_NOT: case OP_NOT3: st[sp - 1] = st[sp - 1] ? 0ull : 1ull; break;  // NULL stays NULL
            case OP_AND: case OP_OR: {
                const int n = in.a;
                bool any_null = false, hit = false;  // hit: a non-NULL false (AND) / true (OR)
                for (int i = sp - n; i < sp; i++) {
                    const bool isn = (nul >> i) & 1u;
                    any_null |= isn;
                    if (!isn && ((st[i] != 0) == (in.op == OP_OR))) hit = true;
                }
                sp -= n - 1;
                const bool rn = !hit && any_null;
                st[sp - 1] = in.op == OP_OR ? (hit ? 1ull : 0ull) : (hit ? 0ull : 1ull);
                nul = rn ? (nul | (1u << (sp - 1))) : (nul & ~(1u << (sp - 1)));
            } break;
            case OP_XOR: {
                sp--;
                const bool n = ((nul >> sp) | (nul >> (sp - 1))) & 1u;
                st[sp - 1] = ((st[sp - 1] != 0) != (st[sp] != 0)) ? 1ull : 0ull;
                nul = n ? (nul | (1u << (sp - 1))) : (nul & ~(1u << (sp - 1)));
            } break;
            case OP_IS_NULL:
                st[sp - 1] = ((nul >> (sp - 1)) & 1u) ? 1ull : 0ull;
                nul &= ~(1u << (sp - 1));
                break;
            case OP_IS_TRUE:
                st[sp - 1] = (!((nul >> (sp - 1)) & 1u) && st[sp - 1] != 0) ? 1ull : 0ull;
                nul &= ~(1u << (sp - 1));
                break;
            case OP_IN: {
                const bool n = (nul >> (sp - 1)) & 1u;
                if (!n) {
                    const int vc = in.c & 0xF;
                    bool found = false;
                    for (int i = 0; i < in.b; i++) found |= cmp_vals(BK_FT_EQ, vc, st[sp - 1], p.cbits[in.a + i]);
                    st[sp - 1] = found ? 1ull : 0ull;
                    if (!found && (in.c >> 4)) nul |= 1u << (sp - 1);  // not found and the list holds a NULL
                }
            } break;
            case OP_IN_SET:
                if (!((nul >> (sp - 1)) & 1u)) {
                    const bool found = in_set_probe(p.cbits[in.a], st[sp - 1], in.c & 0xF);
                    st[sp - 1] = found ? 1ull : 0ull;
                    if (!found && (in.c >> 4)) nul |= 1u << (sp - 1);
                }
                break;
            case OP_SELECT: {   // get_numberic<bool>() of a NULL condition is false
                sp -= 2;
                const bool take_a = !((nul >> (sp - 1)) & 1u) && st[sp - 1] != 0;
                const int src = take_a ? sp : sp + 1;
                st[sp - 1] = st[src];
                nul = ((nul >> src) & 1u) ? (nul | (1u << (sp - 1))) : (nul & ~(1u << (sp - 1)));
            } break;
            case OP_IFNULL:
                sp--;
                if ((nul >> (sp - 1)) & 1u) {
                    st[sp - 1] = st[sp];
                    nul = ((nul >> sp) & 1u) ? (nul | (1u << (sp - 1))) : (nul & ~(1u << (sp - 1)));
                }
                break;
            case OP_MATH:
                if (!((nul >> (sp - 1)) & 1u)) {
                    if (in.a == MF_BIT_COUNT) { st[sp - 1] = (uint64_t)__popcll(st[sp - 1]); break; }   // (UINT64 image in, INT64 image out)
                    const double x = bits_f64(st[sp - 1]);
                    double r;
                    bool null_out = false;
                    switch (in.a) {
                        case MF_ABS: r = x < 0 ? -x : x; break;
                        case MF_FLOOR: r = floor(x); break;
                        case MF_CEIL: r = ceil(x); break;
                        case MF_SQRT: null_out = x < 0; r = sqrt(x); break;
                        case MF_SIGN: st[sp - 1] = (uint64_t)(int64_t)(x > 0 ? 1 : (x < 0 ? -1 : 0)); continue;   // INT64 image
                        case MF_SIN: r = sin(x); break;
                        case MF_COS: r = cos(x); break;
                        case MF_TAN: r = tan(x); break;
                        case MF_ATAN: r = atan(x); break;
                        case MF_ASIN: null_out = x < -1 || x > 1; r = asin(x); break;
                        case MF_ACOS: null_out = x < -1 || x > 1; r = acos(x); break;
                        case MF_COT: { const double s = sin(x), c = cos(x); null_out = fabs(s) < 1e-9; r = __ddiv_rn(c, s); } break;   // float_equal(sin, 0), common.h:1604
                        case MF_LN: null_out = x <= 0; r = log(x); break;
                        default: {   // round half away from zero at `bits` decimals: -::round(-x * base) / base for x < 0
                            const double base = bits_f64(p.cbits[in.b]);
                            r = base > 0 ? (x < 0 ? -__ddiv_rn(round(__dmul_rn(-x, base)), base) : __ddiv_rn(round(__dmul_rn(x, base)), base)) : 0.0;
                        } break;
                    }
                    st[sp - 1] = f64_bits(r);
                    if (null_out) nul |= 1u << (sp - 1);
                }
                break;
            case OP_MATH2: {
                sp--;
                bool n = ((nul >> sp) | (nul >> (sp - 1))) & 1u;
                const double x = bits_f64(st[sp - 1]), y = bits_f64(st[sp]);
                double r = 0;
                if (!n) switch (in.a) {
                    case MF2_FMOD: n = fabs(y) < 1e-9; r = fmod(x, y); break;                                  // mod(): float_equal(rhs, 0) -> NULL
                    case MF2_LOG: n = x <= 0 || y <= 0 || x == 1; r = __ddiv_rn(log(y), log(x)); break;         // log(base, value)
                    case MF2_POW: r = pow(x, y); break;
                    case MF2_GREATEST: r = y > x ? y : x; break;
                    default: r = y < x ? y : x; break;
                }
                st[sp - 1] = f64_bits(r);
                nul = n ? (nul | (1u << (sp - 1))) : (nul & ~(1u << (sp - 1)));
            } break;
            case OP_DATEFN: {
                sp -= in.c - 1;   // datediff's two arguments are at sp - 1 and sp
                bool n = (nul >> (sp - 1)) & 1u;
                if (in.c == 2) n = n || ((nul >> sp) & 1u);
                if (!n) {
                    st[sp - 1] = date_fn(in.a, in.b, st[sp - 1], st[sp]);
                    n = st[sp - 1] == DT_FN_NULL;
                }
                nul = n ? (nul | (1u << (sp - 1))) : (nul & ~(1u << (sp - 1)));
            } break;
            case OP_OUT:
                sp--;
                out[in.a] = st[sp];
                if ((nul >> sp) & 1u) out_null |= 1u << in.a;
                break;
            default: break;
        }
    }
}


}  // namespace bk
