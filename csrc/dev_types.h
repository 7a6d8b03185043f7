// dev_types.h — POD structures shared by the host-side plan lowering (plan.cpp) and the
// sm_90a kernels.  Everything here is passed to kernels BY VALUE (kernel parameter space is a
// constant bank: warp-uniform reads are free), so the structs are small and contain no pointers
// to host memory.
#pragma once
#include <stdint.h>

namespace bk {

// ---- column storage classes (Arrow layout; src/runtime/chunk.cpp:33-92 in the reference) ----
enum SType : int32_t { ST_I32 = 0, ST_U32 = 1, ST_I64 = 2, ST_U64 = 3, ST_F32 = 4, ST_F64 = 5, ST_U8 = 6, ST_BLOB16 = 7,
                       ST_HLL = 8 };   // a RAW HLL sketch of 16400 bytes (MERGE_AGG input of hll_add_agg)

// ---- value classes a device value is held in (the reference evaluates every operator in
//      INT64 / UINT64 / DOUBLE after FunctionManager::complete_fn, src/expr/fn_manager.cpp:316-409) ----
enum VClass : uint8_t { VC_I64 = 0, VC_U64 = 1, VC_F64 = 2 };

constexpr int MAX_COLS = 16;      // distinct input columns one kernel can reference
constexpr int MAX_INSTR = 96;     // bytecode length
constexpr int MAX_CONST = 64;     // constant pool (literals + IN lists + the address of each IN set)
constexpr int MAX_KEYW = 8;       // 64-bit words of a packed GROUP BY key (incl. the null-flag word)
constexpr int MAX_GROUP = 8;      // GROUP BY expressions: encode_exprs_key has 8 null-flag bits
constexpr int MAX_AGG = 12;       // aggregate functions per AggNode
constexpr int MAX_LANES = 26;     // accumulator lanes (8-byte) per group
constexpr int STACK_DEPTH = 12;
constexpr int DIRECT_MAX_AGG = 6; // aggregates the specialised kernels keep in registers
#ifndef BK_DIRECT_THREADS
#define BK_DIRECT_THREADS 512     // threads per CTA of the direct filter+aggregate kernels (one CTA per SM)
#endif
constexpr int DIRECT_THREADS = BK_DIRECT_THREADS;
#ifndef BK_LEAN_THREADS
#define BK_LEAN_THREADS 640       // the lean kernel fits 96 registers: 20 warps per SM fill the 64K-register file (768 threads would spill)
#endif
constexpr int LEAN_THREADS = BK_LEAN_THREADS;
#ifndef BK_LEAN_FX_DEFAULT
#define BK_LEAN_FX_DEFAULT 1      // 1 = the lean kernel's FX variant (fixed-point double sums) is the default; environment BKGPU_LEAN_FX and option lean_fx override
#endif

struct DevCol {
    const void* values;
    const uint8_t* validity;      // Arrow LSB bitmap or nullptr
    int32_t stype;                // SType
    int32_t prim;                 // pb::PrimitiveType of the slot (narrow types are re-narrowed on load)
};

// ---- expression bytecode (postfix).  One instruction = 4 bytes. ----
enum Op : uint8_t {
    OP_END = 0,
    OP_LOAD_COL,     // a = column index, b = 0 | 1 | 2: whole value | {sum | count} half of a 16-byte AVG blob                      -> push value (class by storage), null from bitmap
                     //   b = 3: a FLOAT column's own 4 bytes, zero-extended (hll_add_agg hashes them; the double image may not keep a NaN's bits)
                     //   b = 4: the row index itself (a 16400-byte HLL sketch column: the reader addresses the bytes), null from the bitmap
    OP_CONST,        // a = constant index                    -> push constant
    OP_CAST,         // a = from prim, b = to prim            ExprValue::cast_to (expr_value.h:502-611)
    OP_CMP,          // a = FuncType (EQ..LE), b = VClass     operators.cpp:84-100
    OP_ARITH,        // a = FuncType (ADD/MINUS/MULTIPLIES), b = VClass   operators.cpp:47-50
    OP_DIV_F64,      // NULL on zero divisor                  operators.cpp:65
    OP_MOD,          // b = VClass (I64/U64), NULL on zero    operators.cpp:66-67
    OP_BIT,          // a = FuncType (BIT_AND/OR/XOR/LS/RS)   operators.cpp:70-74 (UINT64)
    OP_BIT_NOT,
    OP_NEG,          // b = VClass                            operators.cpp:30-32
    OP_LOGIC_NOT,    // BOOL in, BOOL out (NULL -> NULL)
    OP_AND,          // a = n children; 3-valued              predicate.h:25-45
    OP_OR,           // a = n children                        predicate.h:81-100
    OP_XOR,
    OP_NOT3,         // NotPredicate: NULL -> NULL
    OP_IS_NULL,
    OP_IS_TRUE,
    OP_IN,           // a = first const, b = count, c = (has_null << 4) | VClass   predicate.cpp:150-189
    OP_OUT,          // a = output register: pop top of stack into out[a]
    OP_SELECT,       // pops [cond, a, b]: cond non-NULL true ? a : b      if_ / case_when (internal_functions.cpp:2351-2388)
    OP_IFNULL,       // pops [a, b]: a NULL ? b : a                           ifnull (internal_functions.cpp:2390-2395)
    OP_MATH,         // a = MathFn on a DOUBLE image, b = constant index (round: 10^bits)   internal_functions.cpp:52-99
    OP_MATH2,        // a = Math2Fn: pops [x, y] DOUBLE images, NULL if either is or outside the domain   internal_functions.cpp:114-127,234-317
    OP_DATEFN,       // a = DateFn, b = mode / unit (datetime.h), c = arguments popped (1, or 2 for datediff); NULL in -> NULL
    OP_IN_SET,       // a = constant holding the set's device address, b = set index in the plan, c = as OP_IN   (in_set.h)
};
enum MathFn : uint8_t { MF_ABS = 0, MF_FLOOR = 1, MF_CEIL = 2, MF_ROUND = 3,
                        // one DOUBLE argument, NULL outside the domain (internal_functions.cpp:101-232); SIGN and BIT_COUNT leave an INT64 image
                        MF_SQRT = 4, MF_SIGN = 5, MF_SIN = 6, MF_ASIN = 7, MF_COS = 8, MF_ACOS = 9, MF_TAN = 10, MF_COT = 11, MF_ATAN = 12, MF_LN = 13, MF_BIT_COUNT = 14 };
enum Math2Fn : uint8_t { MF2_FMOD = 0, MF2_LOG = 1, MF2_POW = 2, MF2_GREATEST = 3, MF2_LEAST = 4 };   // two DOUBLE arguments (OP_MATH2)
struct Instr { uint8_t op, a, b, c; };

struct Program {
    int32_t n_instr;
    int32_t n_out;
    Instr code[MAX_INSTR];
    uint64_t cbits[MAX_CONST];    // constants in their canonical 64-bit image
    uint64_t cnull;               // bit i set = constant i is NULL
};

// ---- aggregate accumulators ----
// Every group owns MAX_LANES 8-byte lanes in the global table.  Lane 0 is always the group's row
// count (COUNT(*) and the "first row seen" marker).  An aggregate names the lane its value
// accumulates in and the lane that counts its non-NULL inputs (0 when the argument cannot be NULL,
// so several aggregates share one counter).
enum AggKind : uint8_t { AG_COUNT_STAR = 0, AG_COUNT = 1, AG_SUM = 2, AG_AVG = 3, AG_MIN = 4, AG_MAX = 5,
                         AG_COUNT_MERGE = 6,     // MERGE_AGG_NODE: counts shipped by the stores are summed (AggFnCall::merge, agg_fn_call.cpp:779-790)
                         AG_HLL = 7,             // hll_add_agg: the value lane holds the group's sketch (index + 1 into GroupTable::hll_regs, 0 = none yet)
                         AG_RB = 8 };            // rb_build_agg: no lane; each non-NULL value appends a key to AggArgs::rb_keys (rb.cu builds the bitmaps)
enum LaneOp : uint8_t { LN_ADD_I64 = 0, LN_ADD_F64 = 1, LN_MIN_I64, LN_MAX_I64, LN_MIN_U64, LN_MAX_U64, LN_MIN_F64, LN_MAX_F64,
                        LN_HLL };                // a sketch reference: never combined as a number (its registers are, by the export / merge kernels)

struct AggSpec {
    uint8_t kind;        // AggKind
    uint8_t vclass;      // class the argument is accumulated in (VClass)
    uint8_t acc_lane;    // value lane (unused for COUNT*)
    uint8_t cnt_lane;    // non-null counter lane (0 = group row count)
    uint8_t arg_out;     // Program output register holding the argument (0xFF = none)
    uint8_t nullable;    // argument can be NULL
    uint8_t out_prim;    // pb::PrimitiveType of the final slot
    uint8_t arg_vclass;  // class the argument VALUE arrives in (converted to `vclass` on update:
                         // AVG does sum += get_numberic<double>(x), agg_fn_call.cpp:525-535)
    uint8_t cnt_owner;   // lanes can be shared by aggregates over the same argument (SUM(x), AVG(x), COUNT(x)):
    uint8_t acc_owner;   // only the owner updates the lane, everyone reads it at finalize
    uint8_t hidden;      // helper accumulator without an output column (the count half of a merged AVG blob)
    uint8_t arg_prim;    // AG_HLL: the argument's type after inference, which sets the bytes hashed (hll_key_bytes); with arg_vclass VC_U64
                         // a FLOAT argument arrives as the column's own 4 bytes (OP_LOAD_COL b = 3), else as its widened double.
                         // BK_HLL: MERGE_AGG over RAW sketches: the argument is the row (OP_LOAD_COL b = 4) of column `hll_col`
    union {
        uint8_t hll_col;
        uint8_t rb_idx;  // AG_RB: which of the plan's rb_build_agg aggregates (0 .. MAX_RB - 1), bits 32-33 of its pair keys
    };
};

struct AggPlan {
    int32_t n_keyw;              // packed key words per group (0 = no GROUP BY)
    int32_t n_group;             // GROUP BY expressions
    int32_t n_agg;
    int32_t n_lanes;             // lanes in use (>= 1)
    uint8_t lane_op[MAX_LANES];  // LaneOp per lane: how partial values combine (AggFnCall::merge)
    AggSpec agg[MAX_AGG];
    // key packing: group expr i occupies key_bits[i] bits at key_shift[i] of word key_word[i];
    // word 0 bit layout is chosen by the host so that a single <=32-bit key + its null flag fits.
    uint8_t key_out[MAX_GROUP];   // Program output register of group expr i
    uint8_t key_word[MAX_GROUP];
    uint8_t key_shift[MAX_GROUP];
    uint8_t key_bits[MAX_GROUP];
    uint8_t key_null_word[MAX_GROUP];
    uint8_t key_null_shift[MAX_GROUP];
    uint8_t key_prim[MAX_GROUP];  // pb::PrimitiveType of the group expression
    int32_t pred_out;             // output register of the filter predicate (-1 = no filter)
    int32_t n_hll;                // AG_HLL aggregates: each adds HLL_ROW_WORDS register words to a group's exported row
};

// ---- specialised ("direct") row evaluation for the canonical shapes: the predicate is a
//      conjunction of `column <cmp> constant`, keys and aggregate arguments are plain columns. ----
struct DirectTerm { uint8_t col, cmp /*FuncType*/, vclass, pad; uint64_t cbits; };
struct DirectPlan {
    int32_t n_terms;              // template NP
    int32_t n_keys;               // template NK (0 or 1)
    int32_t n_vals;               // template NA: distinct aggregate argument columns
    DirectTerm term[4];
    uint8_t key_col[2];
    uint8_t val_col[8];
    uint8_t agg_val[MAX_AGG];     // per aggregate: index into val_col (0xFF = none)
};

// Per value column of the direct kernels, prepared by the host for each batch: which lanes the column
// feeds (SUM / AVG / MIN / MAX over the same column share the load) and its non-NULL counter.
struct ValOps {
    uint8_t n_ops;        // lane operations fed by this column (<= 3)
    uint8_t arg_class;    // VClass the column's canonical image is in
    uint8_t cnt_glob;     // global lane counting non-NULL values (0 = none: shares the row count)
    uint8_t cnt_smem;     // shared lane of that counter in this batch (0xFF = not updated per row)
    uint8_t op[3];        // LaneOp
    uint8_t lane_class[3];
    uint8_t glob_lane[3];
    uint8_t smem_lane[3];
};

// ---- open-addressed group table (global memory; the shared-memory tables use the same layout) ----
struct GroupTable {
    uint32_t* state;     // [cap]   0 empty, 1 busy, 2 full
    uint64_t* keys;      // [n_keyw][cap]
    uint64_t* lanes;     // [n_lanes][cap]
    uint32_t cap_mask;   // cap - 1 (cap is a power of two)
    uint32_t cap_log2;
    uint32_t* n_groups;  // number of occupied slots; n_groups[GT_OCC_OFF + i] = slot of the i-th inserted group (the "occupied list":
                         // re-initialisation, export and result extraction walk the groups that exist, not the table's capacity)
    uint32_t* overflow;  // = n_groups + 1: set when an insert could not find a free slot
    // hll_add_agg: the register arena, one 16384-byte block per (group, AG_HLL aggregate), claimed on a group's first non-NULL value.
    // hll_ctr[0] = blocks claimed, hll_ctr[1] = set when a claim found the arena full (option hll_group_capacity), hll_ctr[2] = set when a
    // MERGE_AGG input value was not a RAW sketch.  nullptr without AG_HLL
    uint8_t* hll_regs;
    uint32_t* hll_ctr;
    uint32_t hll_cap;    // blocks the arena holds
};
constexpr int MAX_RB = 4;             // rb_build_agg aggregates per plan: two key bits name the bitmap's aggregate
constexpr int HLL_ROW_WORDS = 2048;   // one sketch's 16384 registers as 64-bit words of an exported group row
constexpr uint64_t HLL_LANE_BUSY = ~0ull;          // a sketch lane while its block is being claimed and zeroed
constexpr uint64_t HLL_LANE_FULL = ~0ull - 1;      // a sketch lane whose claim found the arena full (the request fails with ETOOBIG)
constexpr int GT_TICKET = 6;    // word 6 of the counter block: CTAs of the running lean launch that have finished (fused_extract, agg_kernels.cuh); 0 between launches
constexpr int GT_FX_EXACT = 7;  // word 7 of the counter block: double values the lean kernel's FX variant could not put on its fixed-point grid (agg_direct.cuh)
constexpr int GT_OCC_OFF = 8;   // words 0-7 of the counter block: groups, overflow, result cursor, merge info, rows passed (u64), ticket, FX exact:
                                // one 32-byte device-to-host copy brings every counter of a finished request back

}  // namespace bk
