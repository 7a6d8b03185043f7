/*
 * bkgpu.h — C ABI of the GPU execution path for BaikalDB's analytical
 * scan -> filter -> aggregate / join / sort subtree.
 *
 * The reference has no FFI for this path: operators are C++ virtuals
 *     ExecNode::init / open / get_next / close
 *         /root/reference/include/exec/exec_node.h:88,140-153
 * instantiated by the switch in ExecNode::create_exec_node
 *         /root/reference/src/exec/exec_node.cpp:396-490
 * and driven by Region::select (src/store/region.cpp:3069-3119) on the store and
 * PacketNode::open (src/exec/packet_node.cpp:855-897) on the db.  A maintainer
 * adds one `GpuExecNode : ExecNode` (see INTEGRATION.md) whose four virtuals
 * forward to the entry points below; everything behind them is CUDA for sm_90a.
 *
 * Conventions (mirroring the reference's: negative int + message, no exceptions):
 *   - every int-returning call gives 0 on success and a negative BKGPU_E* code on
 *     failure; bkgpu_last_error() returns the message for the plan (or for the
 *     calling thread when the plan pointer is NULL).
 *   - one plan = one host thread + one CUDA stream (the reference runs one
 *     bthread per plan fragment, src/exec/agg_node.cpp:447-485).
 *   - threads: different plans, and different bkgpu_dict handles, may be driven
 *     from different host threads at the same time — pageable pushes and plans on
 *     different devices included (the copy workers, the device-buffer caches and
 *     the resident regions are process-wide and shared safely; concurrent pageable
 *     pushes take turns on the copy workers).  One plan takes one call at a time;
 *     the exception is bkgpu_cancel, which may come from any thread.  Calls that
 *     need no plan (explain, regions, memory helpers) may come from any thread;
 *     bkgpu_last_error(NULL) is the calling thread's own last message.
 *   - there is NO CPU fallback: without a usable CUDA device every call that
 *     needs one fails with BKGPU_ENODEV.
 */
#ifndef BKGPU_H_
#define BKGPU_H_

#include <stddef.h>
#include <stdint.h>
#include "bkgpu_plan.h"

#ifdef __cplusplus
extern "C" {
#endif

#define BKGPU_OK          0
#define BKGPU_EINVAL     -1   /* malformed plan / argument                          */
#define BKGPU_EUNSUPPORTED -2 /* well-formed but outside the GPU path (e.g. STRING) */
#define BKGPU_ENODEV     -3   /* no CUDA device / CUDA runtime error                */
#define BKGPU_ENOMEM     -4   /* device or pinned allocation failed                 */
#define BKGPU_ESTATE     -5   /* call out of order (push before open, ...)          */
#define BKGPU_ECANCELLED -6   /* bkgpu_cancel() was observed (RuntimeState::is_cancelled) */
#define BKGPU_ETOOBIG    -7   /* group table overflow; ER_TOO_BIG_SELECT analogue
                                 (src/runtime/runtime_state.cpp:289-311)            */
#define BKGPU_ENCCL      -8   /* NCCL unavailable or a collective failed            */

typedef struct bkgpu_plan bkgpu_plan; /* opaque; owns device state */

/*
 * One column of a batch, Arrow layout (the layout Chunk builds for the
 * vectorized engine: /root/reference/src/runtime/chunk.cpp:33-92 —
 * INT8/16/32,TIME -> int32; INT64 -> int64; UINT8/16/32,TIMESTAMP,DATE -> uint32;
 * UINT64,DATETIME -> uint64; FLOAT -> float32; DOUBLE -> float64; BOOL -> uint8 here).
 * `validity` is an LSB-first bitmap (1 = valid) or NULL when the column has no NULLs.
 * Columns are named the way the reference names Arrow fields: "<tuple>_<slot>"
 * (include/expr/slot_ref.h:72-82).
 */
typedef struct bkgpu_column {
    int32_t        tuple_id;
    int32_t        slot_id;
    int32_t        prim_type;   /* bkgpu_primitive_type == pb::PrimitiveType value    */
    int32_t        elem_size;   /* bytes per value; 0 = derive from prim_type; 16 for
                                   the AVG intermediate {double sum; int64 count}
                                   (include/expr/agg_fn_call.h:41-47)                  */
    const void*    values;
    const uint8_t* validity;
    int64_t        length;
} bkgpu_column;

/* Per-plan counters (the fields Region::select copies into the response,
 * src/store/region.cpp:3140-3143, plus device timings for the bench). */
typedef struct bkgpu_stats {
    int64_t rows_scanned;        /* RuntimeState::num_scan_rows                       */
    int64_t rows_filtered;       /* RuntimeState::num_filter_rows (dropped by filter) */
    int64_t rows_returned;
    int64_t kernel_launches;     /* kernels of this library launched for the plan     */
    int64_t h2d_bytes;
    int64_t d2h_bytes;
    double  main_kernel_ms;      /* summed device time of the dominant kernel          */
    int64_t main_kernel_launches;
    int64_t main_kernel_bytes;   /* algorithmic bytes those launches covered          */
    double  collective_ms;       /* device time inside the NCCL exchange + merge      */
    char    main_kernel_name[64];
} bkgpu_stats;

/* ---- library ---------------------------------------------------------- */
const char* bkgpu_version(void);
int   bkgpu_device_count(void);                /* >=0, or BKGPU_ENODEV               */
const char* bkgpu_last_error(bkgpu_plan* plan_or_null);

/* Host-only: parse + type-infer + lower a plan without touching CUDA.  Writes a
 * human-readable description of the lowered device program into `text`.
 * Mirrors what ExecNode::create_tree + expr type_inferer do at plan time
 * (src/exec/exec_node.cpp:347-394, src/expr/scalar_fn_call.cpp:40-120). */
int   bkgpu_plan_explain(const uint8_t* plan_desc, size_t len, char* text, size_t text_len);

/* ---- operator lifecycle: ExecNode::init/open/get_next/close ----------- */
/* ExecNode::init(const pb::PlanNode&) for the whole subtree (exec_node.h:88).
 * `nccl_comm_or_null`: an ncclComm_t to merge per-GPU partial results inside
 * bkgpu_finish (regions -> one set per GPU; src/physical_plan/separate.cpp:249-258). */
int   bkgpu_init(bkgpu_plan** out, const uint8_t* plan_desc, size_t len,
                 int device, void* nccl_comm_or_null);
/* Tunables, before open:
 *   "stream"               cudaStream_t (as int64) the plan launches on (default: its own stream)
 *   "group_capacity_log2"  slots of the global group table (default 20); overflow -> BKGPU_ETOOBIG
 *   "smem_capacity_log2"   slots of the per-CTA shared table (-1 = chosen per batch, 0 = none)
 *   "batch_capacity"       rows per bkgpu_get_next batch (RuntimeState::row_batch_capacity)
 *   "chunk_rows"           rows per host->device staging chunk of a host push
 *   "partial_capacity"     groups per rank in the exported partial state (a plan with hll_add_agg ships 16 KB of registers per group and sketch)
 *   "rb_pair_capacity"     keys the rb_build_agg pair buffer holds: one per row and rb_build_agg with a non-NULL value until it is sorted
 *                          and deduplicated, which happens whenever it could overflow (default 2^27; 16 bytes of device memory each, the sort
 *                          needs a second buffer, and its look-back scratch takes 1 KB per 3072 keys and active 8-bit digit; 1024 .. 2^30 - 1);
 *                          more distinct (group, value) pairs -> BKGPU_ETOOBIG naming this option
 *   "hll_group_capacity"   sketches the hll_add_agg register arena holds: one per group and hll_add_agg aggregate that receives a non-NULL
 *                          value, 16 KB of device memory each (default 4096 = 64 MB, at most 2^20); more -> BKGPU_ETOOBIG naming this option
 *   "region_base"          arrival index of this plan's first row: ORDER BY ties across GPUs break by (region, row)
 *   "repartition"          with a communicator: groups are hash-partitioned across the ranks by one all-to-all (ncclSend/ncclRecv)
 *                          instead of gathered everywhere; each rank then returns only the groups it owns (high-cardinality GROUP BY)
 *   "force_generic" / "no_lean" / "no_lean_nulls" / "no_lean_mm" / "no_fused_probe"   pin the kernel variant (tests, A/B measurements)
 *   "scalar_tma"           0 = COUNT(*) WHERE int32 <cmp> c takes the LDG kernel instead of the TMA-staged one (csrc/scalar_tma.cu; default 1)
 *   "star_expand_capacity" (tests) first capacity, in row-id tuples, of a star join's expansion pass over a dimension with duplicate keys
 *                          (0 = twice the pass's input); a pass that outgrows it is counted, grown to the exact count and run again
 *   "blocking_sync"        the wait for a request's result: 0 spins (cudaStreamSynchronize), 1 sleeps on a blocking-sync event, -1 (default) sleeps only
 *                          when several ranks share a small CPU budget (ranks > 1 and budget < 4 CPUs per rank)
 *   "lean_fx"              (default 1; environment BKGPU_LEAN_FX) SUM / AVG over DOUBLE columns in the lean kernel accumulate as fixed-point
 *                          limbs with native 32-bit shared-memory atomics (csrc/fx.h: every value keeps M - 14 significant bits, where
 *                          M = 62 - ceil(log2(rows one CTA adds)): 28 bits for a 100M-row batch on 132 SMs, 26 bits from about 277M
 *                          rows; typically 1e-13 of sum|x|; 0 = IEEE adds through 64/128-bit compare-and-swap loops); bkgpu_stats.main_kernel_name says
 *                          "k_agg_group_lean_fx" when a batch ran that way */
int   bkgpu_set_option(bkgpu_plan*, const char* key, int64_t value);
/* ExecNode::open(RuntimeState*) (exec_node.h:140): allocate tables. */
int   bkgpu_open(bkgpu_plan*);
/* child->get_next() inverted: feed one column batch of the scan tuple the columns
 * name.  HOST buffers (on_device == 0) are borrowed for the duration of the call: every host-to-device copy has
 * read them when bkgpu_push returns (pinned or pageable alike).  on_device != 0 means `values`/`validity` are
 * device pointers on the plan's device; the kernels read them asynchronously on the plan's stream, so DEVICE
 * buffers must stay valid and unmodified until bkgpu_finish has returned (or until work the caller orders after
 * the plan's stream has run).
 * Joins: a batch belongs to the table whose tuple its columns name.  Every batch of the build side (a two-table join's
 * outer child; every dimension of a star join) is retained and must come before the first batch of the probe side (the
 * inner child; the star join's fact table): a build-side batch after that returns BKGPU_ESTATE.  A caller that pulls
 * its children in order puts the fact scan last. */
int   bkgpu_push(bkgpu_plan*, const bkgpu_column* cols, int ncols, int64_t nrows, int on_device);
/* End of input: drain, run the cross-GPU merge when a communicator was given,
 * finalize aggregates (AggFnCall::finalize, src/expr/agg_fn_call.cpp:927-990). */
int   bkgpu_finish(bkgpu_plan*);
/* ExecNode::get_next(RuntimeState*, RowBatch*, bool* eos) (exec_node.h:143): up to
 * *ncols (in: capacity of out_cols, out: columns written) columns of the next result
 * batch; buffers are owned by the plan until the next call / close. */
int   bkgpu_get_next(bkgpu_plan*, bkgpu_column* out_cols, int* ncols, int64_t* nrows, int* eos);
/* Re-arm an executed plan for the next request of the same fragment (the reference caches plans of
 * prepared statements; a maintainer may instead init/close per request): tables are cleared,
 * allocations and streams kept.  Valid after open or finish. */
int   bkgpu_reset(bkgpu_plan*);
/* state->cancel(); polled between launches like RuntimeState::is_cancelled.  May be called from any thread while another thread
 * drives the plan.  After it, the plan's bkgpu_push / bkgpu_finish give BKGPU_ECANCELLED and bkgpu_get_next gives eos with no rows,
 * until bkgpu_reset re-arms the plan. */
void  bkgpu_cancel(bkgpu_plan*);
/* ExecNode::close + destroy_tree. */
void  bkgpu_close(bkgpu_plan*);
int   bkgpu_get_stats(bkgpu_plan*, bkgpu_stats* out);

/* Device buffers (and the mapped host buffers GROUP BY results land in) of closed plans are kept in a process-wide cache and handed
 * to the next plan (a store opens one plan per request; cudaMalloc / cudaFree of the group table would cost milliseconds each).  This
 * returns the cached memory to the driver.
 * Environment BKGPU_NO_ALLOC_CACHE=1 disables the cache. */
void  bkgpu_release_cache(void);

/* ---- date/time literals ----
 * The text of a literal as the image the plan compares against: ExprValue::cast_to from STRING (include/common/expr_value.h:534-573
 * -> str_to_datetime / str_to_time, src/common/datetime.cpp:149-263,477-560), for a binding that folds `col >= '2024-01-31'`
 * itself.  prim_type: BK_DATETIME, BK_TIMESTAMP, BK_DATE or BK_TIME; *image: the 64-bit canonical image (TIMESTAMP / DATE
 * zero-extended, TIME sign-extended).  Text that is not a date gives the zero image, as in the reference.  Needs no GPU. */
int   bkgpu_parse_datetime(const char* text, size_t length, int prim_type, uint64_t* image);
/* ExprValue::cast_to (include/common/expr_value.h:502-611) between two non-STRING primitive types, on canonical images — the
 * conversion plan compilation applies to literals (DATE <-> DATETIME <-> TIMESTAMP in the reference's fixed UTC+8 zone included).
 * BKGPU_EUNSUPPORTED for a TIME source with another date/time target (relative to the current date in the reference). */
int   bkgpu_cast_image(uint64_t image, int from_prim, int to_prim, uint64_t* out);

/* ---- HyperLogLog sketches ----
 * hll_add_agg returns a column of prim_type BK_HLL and elem_size 16400: the reference's RAW sketch (hll_row_init, src/common/
 * hll_common.cpp:834-842): "HYLL", encoding byte 255, three zero bytes, 8 bytes of cached cardinality (bit 7 of the last one set = not
 * cached), then 16384 one-byte registers.  bkgpu_hll_estimate is hll_estimate (hll_common.cpp:523-600) over such a sketch: the cached
 * value when it is valid, else the histogram estimator; the sketch itself is not modified.  BKGPU_EINVAL for anything but a RAW sketch
 * of 16400 bytes.  Needs no GPU.
 * MERGE_AGG of hll_add_agg takes the stores' sketches as input columns of the same type and size (RAW only: any other value fails the push
 * with BKGPU_EINVAL, or bkgpu_finish when the column is in device memory). */
int   bkgpu_hll_estimate(const uint8_t* sketch, size_t len, uint64_t* estimate);

/* ---- Roaring bitmaps ----
 * rb_build_agg returns a column of prim_type BK_BITMAP (21) with elem_size -1 and no validity bitmap (a group whose values were all NULL
 * holds the empty bitmap, 3a300000 00000000).  Its values are variable-length, in Arrow's large_binary layout in one buffer: `length + 1`
 * int64 offsets (the first 0), followed directly by the bytes; value r is bytes [offsets[r], offsets[r + 1]).  Each value is the
 * reference's bitmap of the group's values' low 32 bits after runOptimize(), in CRoaring's portable serialization (v0.2.66).
 * The buffer stays valid until the next bkgpu_get_next, bkgpu_reset or bkgpu_close. */

/* ---- resident regions (the column store / parquet cache analogue, include/column/file_manager.h:252-272) ----
 * A region's columns are copied to HBM once (host or device source) and stay there across queries, keyed by
 * (device, region_id); bkgpu_push_region feeds them to a plan exactly like bkgpu_push(..., on_device = 1) — a query
 * over a resident region moves no input over PCIe.  Registering an id again replaces the region.
 * bkgpu_region_info gives its rows and the bytes of its values and validity bitmaps.  A malformed column, an unknown id (never
 * registered, or evicted) give BKGPU_EINVAL.
 * Lifetime: the kernels of a plan that pushed a region read its device buffers asynchronously until that plan's bkgpu_finish has
 * returned, as with any device batch.  A region must not be evicted or registered again while such a plan has not returned from
 * bkgpu_finish (or been closed); other region ids may be registered and evicted at any time, from any thread. */
int   bkgpu_region_register(int device, int64_t region_id, const bkgpu_column* cols, int ncols, int64_t nrows, int on_device);
int   bkgpu_region_evict(int device, int64_t region_id);
int   bkgpu_region_info(int device, int64_t region_id, int64_t* nrows, size_t* bytes);
int   bkgpu_push_region(bkgpu_plan*, int64_t region_id);

/* ---- per-GPU partial state (MERGE_AGG / merge-sort on the db side) ---- */
/* After bkgpu_finish on a plan WITHOUT a communicator the caller may move the
 * partial state itself (e.g. torch.distributed all_gather): export gives a device
 * buffer of `*bytes` bytes (fixed per plan: see bkgpu_partial_capacity), merge
 * folds `nranks` such buffers (AggFnCall::merge, agg_fn_call.cpp:719-822;
 * SelectManagerNode merge sort, select_manager_node.cpp:50-51) and re-finalizes. */
int   bkgpu_partial_capacity(bkgpu_plan*, size_t* bytes);
int   bkgpu_partial_export(bkgpu_plan*, void* dev_dst, size_t bytes);
int   bkgpu_partial_merge(bkgpu_plan*, const void* dev_src, size_t bytes_per_rank, int nranks);

/* ---- NCCL plumbing (dlopen'ed libnccl.so.2; one communicator per process) */
int   bkgpu_nccl_unique_id(uint8_t id_out[128]);
int   bkgpu_nccl_comm_create(void** comm_out, const uint8_t id[128], int nranks, int rank, int device);
void  bkgpu_nccl_comm_destroy(void* comm);

/* ---- host / device memory helpers for adapters and the bench ---------- */
void* bkgpu_host_alloc(size_t bytes);          /* pinned; NULL on failure            */
void  bkgpu_host_free(void* p);
void* bkgpu_device_alloc(int device, size_t bytes);
void  bkgpu_device_free(int device, void* p);
int   bkgpu_memcpy_h2d(int device, void* dst, const void* src, size_t bytes);
int   bkgpu_memcpy_d2h(int device, void* dst, const void* src, size_t bytes);

/* Synthetic column generator on the device (SURVEY.md §8d): counter-based, keyed by
 * (seed, column_id, absolute row index) so any shard of any table is reproducible
 * and bit-identical to baikaldb_b200/datagen.py.  dist: 0 = uniform int in [lo,hi) (int32/
 * int64 by prim_type), 1 = uniform double in [0,1), 2 = approx-normal double
 * (Irwin-Hall 4) * scale, 3 = full-range int64, 4 = permutation of [0,n) (int32). */
int   bkgpu_gen_column(int device, void* dev_dst, int32_t prim_type, int32_t dist,
                       uint64_t seed, uint32_t column_id, int64_t row0, int64_t nrows,
                       int64_t lo, int64_t hi, double scale);

/* ---- order-preserving dictionary of STRING columns (csrc/dict.cu) ----
 * The device counterpart of baikaldb_b200/dictionary.py's encoder: one comparison domain (the columns that are compared with each other,
 * e.g. the two sides of a join condition) -> its sorted distinct values and, per column, the INT32 rank of every row's value in them.
 * Order: unsigned bytes, a proper prefix first (std::string::compare; Arrow's sort of binary values).  A NULL gets code 0 and a clear
 * validity bit.  Needs no plan.
 *
 * A column in Arrow's large_binary layout, every buffer in device memory on the handle's device: value r is bytes
 * [offsets[r], offsets[r + 1]) of `data`; `offsets` has length + 1 entries and need not start at 0 (a sliced array: pass the buffer
 * advanced by the slice offset).  `validity`: LSB-first bitmap, row r at bit validity_offset + r, or NULL when no value is NULL.
 * NOT validated: the device buffers themselves.  Offsets are trusted to be non-decreasing and inside `data`, as device batches of
 * bkgpu_push are trusted; `data` must be non-NULL even when every value is empty. */
typedef struct bkgpu_binary_column {
    const int64_t* offsets;
    const uint8_t* data;
    const uint8_t* validity;
    int64_t        validity_offset;
    int64_t        length;
} bkgpu_binary_column;

typedef struct bkgpu_dict bkgpu_dict;   /* opaque; owns the dictionary and the codes in device memory */

/* Build the dictionary of `ncols` columns on `device`, on `stream_or_null` (a cudaStream_t; NULL: the handle's own stream).  The columns
 * are read during the call only.  hash_bits: 0 for the full 64-bit hash; 1 .. 63 keep only that many bits (tests: forces hash collisions,
 * which the byte comparison resolves).  BKGPU_EINVAL: out or cols NULL, ncols < 1, a negative length or validity offset, NULL offsets or
 * data, a bad device index; BKGPU_ENODEV: no device; BKGPU_EUNSUPPORTED: more than 2^30 rows in all, or 2^31 distinct values (the host
 * encoder's limit); BKGPU_ENOMEM.  The message of a failure: bkgpu_last_error(NULL). */
int   bkgpu_dict_build(bkgpu_dict** out, int device, void* stream_or_null, const bkgpu_binary_column* cols, int ncols, int hash_bits);
/* distinct values, and their bytes in all */
int   bkgpu_dict_size(bkgpu_dict*, int64_t* n_values, int64_t* n_bytes);
/* the sorted values in large_binary layout: n_values + 1 offsets from 0, and n_bytes bytes; host (on_device = 0) or device destinations.
 * Returns when the copy is done. */
int   bkgpu_dict_copy(bkgpu_dict*, int64_t* offsets, uint8_t* bytes, int on_device);
/* column `column`'s codes (length int32, device) and validity bitmap from bit 0 ((length + 7) / 8 bytes, device; NULL: not written);
 * *null_count (may be NULL) = its NULLs.  Returns when the codes are written. */
int   bkgpu_dict_codes(bkgpu_dict*, int column, int32_t* codes, uint8_t* validity, int64_t* null_count);
void  bkgpu_dict_free(bkgpu_dict*);

#ifdef __cplusplus
}
#endif
#endif /* BKGPU_H_ */
