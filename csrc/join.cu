// join.cu — host path of the hash join (K4): the retained build sides and their indexes, the two-table probe (fused into the lean
// aggregate, gather, general), the outer-join tail, the join that returns rows, and the star join's build and probe.
#include <string.h>
#include <algorithm>
#include <vector>
#include "api_state.h"

// every plan column of the joined row: the build sides' retained columns and the probe batch's (nullptr: the outer-join tail, whose
// probe-side columns are never read — row = -1 is NULL)
static std::vector<DevCol> join_cols(const bkgpu_plan* p, const DevCol* probe_cols) {
    const Compiled& c = p->c;
    std::vector<DevCol> all(c.cols.size());
    for (size_t i = 0; i < c.cols.size(); i++) {
        all[i].stype = prim_storage(c.cols[i].prim); all[i].prim = c.cols[i].prim;
        if (c.col_side[i] > 0) all[i] = store_col(p->join.side[c.col_side[i] - 1].store, i);
    }
    if (probe_cols) for (size_t w = 0; w < p->join.probe_map.size(); w++) all[(size_t)p->join.probe_map[w]] = probe_cols[w];
    return all;
}

// a 4-byte device counter, read once the stream has reached it
static int read_u32(bkgpu_plan* p, const uint32_t* dev, uint32_t* out) {
    CK(p, cudaMemcpyAsync(out, dev, 4, cudaMemcpyDeviceToHost, p->stream));
    CK(p, cudaStreamSynchronize(p->stream));
    return BKGPU_OK;
}
// a pass whose output can outgrow its buffer: `run(cap)` sizes the buffer for `cap` items and launches the pass, which writes at most
// `cap` of them and counts all of them in `cursor`; a pass that found more is rerun once, with the buffer grown to the count
template <class Run>
static int run_counted(bkgpu_plan* p, uint64_t cap, const uint32_t* cursor, uint32_t* found, Run run) {
    for (int attempt = 0; attempt < 2; attempt++) {
        int rc;
        if ((rc = run(cap)) || (rc = read_u32(p, cursor, found))) return rc;
        if (*found <= cap) break;
        cap = *found;
    }
    return BKGPU_OK;
}

JoinArgs join_args(const bkgpu_plan* p, bool tail) {
    const Compiled& c = p->c;
    const JoinSide& s = p->join.side[0];
    JoinArgs a; memset(&a, 0, sizeof a);
    a.enabled = 1; a.keys = s.jt_keys; a.rows = s.jt_rows; a.cap_mask = s.jt_mask;
    a.probe_col = c.probe_key_col; a.probe_prim = c.cols[(size_t)c.probe_key_col].prim; a.cast_prim = c.join_key_prim;
    a.join_type = c.join_type; a.matched = c.join_type == BK_INNER_JOIN ? nullptr : p->join.matched; a.n_build = s.store.rows;
    a.tail = tail ? 1 : 0;
    return a;
}

// ---- retain the build (outer / driver) table, build its indexes at the first probe batch ----
// `side`: the Compiled::col_side value of this table's columns (1 for the two-table join, 1 + d for dimension d of a star join)
static int join_retain_build(bkgpu_plan* p, int side, const bkgpu_column* cols, int ncols, int64_t nrows, int on_device) {
    const Compiled& c = p->c;
    JoinSide& s = p->join.side[side - 1];
    if (p->join.built) return p->fail(BKGPU_ESTATE, "build-side rows arrived after probing started (the reference fetches the whole driver table first, join_node.cpp:920-1022)");
    const size_t nc = c.cols.size();
    std::vector<ColRef> want; std::vector<int> idx;
    for (size_t i = 0; i < nc; i++) if (c.col_side[i] == side) { want.push_back(c.cols[i]); idx.push_back((int)i); }
    std::vector<const bkgpu_column*> bound;
    int rc = bind_columns(p, want, cols, ncols, nrows, bound);
    if (rc) return rc;
    if (s.store.rows + nrows > 0xFFFFFFF0ll) return p->fail(BKGPU_EUNSUPPORTED, "build side larger than 2^32 rows");
    if ((rc = store_retain(p, s.store, s.store.rows + nrows))) return rc;
    for (size_t w = 0; w < want.size(); w++) {
        if ((rc = store_append(p, s.store, (size_t)idx[w], *bound[w], nrows, on_device))) return rc;
        if (on_device) p->stats.kernel_launches++;   // (the unpack kernel)
    }
    s.store.rows += nrows;
    return BKGPU_OK;
}

// Fused probe (JoinProbe in agg.h): usable when the only build-side column the aggregate reads is its 4-byte GROUP BY
// key and the probe key is a 32-bit integer column whose cast to the comparison type keeps the canonical image.
static int join_compose_probe(bkgpu_plan* p, uint32_t* flag) {
    const Compiled& c = p->c;
    JoinState& j = p->join;
    const JoinSide& s = j.side[0];
    j.jp = JoinProbe{};
    if (!c.jfast || !c.jfast->has_direct || c.jfast->direct.n_keys != 1) return BKGPU_OK;
    const Compiled& f = *c.jfast;
    const size_t kpos = (size_t)f.direct.n_terms;
    int attr_main = -1;
    for (size_t i = 0; i < f.direct_cols.size(); i++) {
        const int m = c.jfast_of_main[(size_t)f.direct_cols[i]];
        if (c.col_side[(size_t)m] != 1) continue;
        if (i != kpos) return BKGPU_OK;   // a predicate or an aggregate argument comes from the build side: gather path
        attr_main = m;
    }
    if (attr_main < 0) return BKGPU_OK;
    const int ast = prim_storage(c.cols[(size_t)attr_main].prim);
    if ((ast != ST_I32 && ast != ST_U32) || (c.cols[(size_t)attr_main].prim != BK_INT32 && c.cols[(size_t)attr_main].prim != BK_UINT32)) return BKGPU_OK;
    const int pp = c.cols[(size_t)c.probe_key_col].prim, ct = c.join_key_prim;
    const bool ident = (pp == BK_INT32 && (ct == BK_INT32 || ct == BK_INT64)) || (pp == BK_UINT32 && (ct == BK_UINT32 || ct == BK_UINT64 || ct == BK_INT64));
    if (!ident) return BKGPU_OK;
    int rc;
    JoinProbe jp{};
    jp.mode = s.jf.mode; jp.key_signed = pp == BK_INT32 ? 1 : 0;
    jp.dense_min = s.jf.dense_min; jp.dense_size = s.jf.dense_size; jp.bias = s.jf.bias; jp.packed_mask = s.jf.packed_mask;
    if (jp.mode == 1) {
        if ((rc = ensure_buf(p, (void**)&j.jp_attr, &j.jp_attr_cap, (size_t)jp.dense_size * 4))) return rc;
        jp.attr = j.jp_attr;
        jp.present = (uint64_t)s.store.rows == jp.dense_size ? nullptr : s.jf.dense;   // unique, NULL-free keys filling the range: every key exists
    } else {
        if ((rc = ensure_buf(p, (void**)&j.jp_packed, &j.jp_packed_cap, ((size_t)jp.packed_mask + 1) * 8))) return rc;
        jp.packed = j.jp_packed;
    }
    CK(p, launch_join_compose(s.jf, (const uint32_t*)s.store.cols[(size_t)attr_main].vals, j.jp_attr, j.jp_packed, flag, p->stream));
    p->stats.kernel_launches++;
    j.jp = jp; j.jp_key_pos = (int)kpos;   // (the caller drops it again when `flag` comes back set)
    return BKGPU_OK;
}

// validity bitmaps of the side's retained columns that some batch delivered NULLs for (store_col reads no bitmap of the others)
static int join_pack_validity(bkgpu_plan* p, JoinSide& s) {
    int rc;
    DevCol d;
    for (size_t i = 0; i < s.store.cols.size(); i++) {
        if (!s.store.cols[i].nullable) continue;
        if ((rc = store_pack(p, s.store, i, s.store.rows, 16, nullptr, &d))) return rc;
        p->stats.kernel_launches++;
    }
    return BKGPU_OK;
}

// The unique-key index of side `s` (FK -> PK fast path): a dense array when the key range is small, else a packed table for keys of at most
// 32 bits.  s.jf.mode stays 0 when neither fits or a key repeats.  `compose`: the two-table join's fused probe is composed behind the build,
// so that its flag comes back in the same round trip.
static int join_build_index(bkgpu_plan* p, JoinSide& s, const DevCol& key, int cast_prim, bool compose) {
    JoinState& j = p->join;
    int rc;
    s.jf = JoinFast{};
    if (s.store.rows <= 0) return BKGPU_OK;
    bool retry_measured = false;
again:
    const int cls = host_prim_class(cast_prim);
    const uint64_t bias = cls == VC_I64 ? 0x8000000000000000ull : 0ull;
    if ((rc = ensure_buf(p, (void**)&j.scratch, &j.scratch_cap, 64))) return rc;
    uint64_t* mm = j.scratch; uint32_t* dup = (uint32_t*)(j.scratch + 2);
    // the key range: measured (one pass over the keys + a round trip), or — when this plan has built before — the range it saw then,
    // checked by the build kernel itself (a key outside it raises a flag and the build is redone with a measured range)
    uint64_t h_mm[2];
    bool guessed = s.learned && !retry_measured;
    if (guessed) { h_mm[0] = s.learn_min; h_mm[1] = s.learn_max; }
    else {
        CK(p, launch_join_minmax(key, key.prim, cast_prim, s.store.rows, bias, mm, p->stream));
        CK(p, cudaMemcpyAsync(h_mm, mm, 16, cudaMemcpyDeviceToHost, p->stream));
        CK(p, cudaStreamSynchronize(p->stream));
        p->stats.kernel_launches++;
    }
    JoinFast jf{}; jf.bias = bias;
    const uint64_t range = h_mm[1] >= h_mm[0] ? h_mm[1] - h_mm[0] + 1 : 0;
    const int kb = storage_bytes(prim_storage(cast_prim));
    if (range > 0 && range <= (uint64_t)4 * (uint64_t)s.store.rows + 1024 && range <= (1ull << 30)) {
        jf.mode = 1; jf.dense_min = h_mm[0]; jf.dense_size = range;
        if ((rc = ensure_buf(p, (void**)&s.jf_dense, &s.jf_dense_cap, (size_t)range * 4))) return rc;
        jf.dense = s.jf_dense;
    } else if (kb <= 4) {
        uint32_t pc = 1024; while ((int64_t)pc < 2 * s.store.rows) pc <<= 1;
        jf.mode = 2; jf.packed_mask = pc - 1;
        if ((rc = ensure_buf(p, (void**)&s.jf_packed, &s.jf_packed_cap, (size_t)pc * 8))) return rc;
        jf.packed = s.jf_packed;
    }
    if (jf.mode) {
        CK(p, launch_join_build_fast(key, key.prim, cast_prim, s.store.rows, jf, s.jf_dense, s.jf_packed, dup, p->stream));
        p->stats.kernel_launches += 1;
        s.jf = jf;
        if (compose && (rc = join_compose_probe(p, dup + 1))) return rc;   // enqueued behind the build: all flags come back in one round trip
        uint32_t h_flags[3] = {0, 0, 0};
        CK(p, cudaMemcpyAsync(h_flags, dup, 12, cudaMemcpyDeviceToHost, p->stream));
        CK(p, cudaStreamSynchronize(p->stream));
        if (h_flags[2] && guessed) { retry_measured = true; goto again; }   // this run's keys left the learned range
        if (h_flags[0]) { s.jf = JoinFast{}; j.jp = JoinProbe{}; }   // duplicate build keys: not a PK, the general probe runs
        else if (h_flags[1]) j.jp = JoinProbe{};
        s.learned = true; s.learn_min = h_mm[0]; s.learn_max = h_mm[1];
    } else if (guessed) { retry_measured = true; goto again; }   // (the learned range no longer fits this row count)
    return BKGPU_OK;
}

static int join_build_table(bkgpu_plan* p) {
    const Compiled& c = p->c;
    JoinState& j = p->join;
    JoinSide& s = j.side[0];
    int rc;
    if ((rc = join_pack_validity(p, s))) return rc;
    j.built = true; s.jt_generic = false;   // the multimap of the general probe is built on first use (join_generic_table)
    // ---- FK -> PK fast path: are the build keys unique, and is their range dense or their type <= 32 bits? ----
    s.jf = JoinFast{}; j.jp = JoinProbe{};
    bool build_nulls = false;
    for (const RowStore::Col& col : s.store.cols) if (col.nullable) build_nulls = true;   // gathered columns must be NULL-free
    if (!c.jfast || c.join_type == BK_FULL_JOIN || build_nulls) return BKGPU_OK;
    return join_build_index(p, s, store_col(s.store, (size_t)c.build_key_col), c.join_key_prim, true);
}

// the multimap of side `s` (duplicate build keys, the general probe): open addressing from the cast key image to the build row
static int join_build_multimap(bkgpu_plan* p, JoinSide& s, const DevCol& key, int cast_prim) {
    int rc;
    uint32_t cap = 1024;
    while ((int64_t)cap < 2 * s.store.rows) cap <<= 1;
    dev_free(p, s.jt_keys); dev_free(p, s.jt_rows); s.jt_keys = nullptr; s.jt_rows = nullptr;
    if ((rc = dev_alloc(p, (void**)&s.jt_keys, (size_t)cap * 8))) return rc;
    if ((rc = dev_alloc(p, (void**)&s.jt_rows, (size_t)cap * 4))) return rc;
    s.jt_mask = cap - 1;
    CK(p, launch_join_build(key, key.prim, cast_prim, s.store.rows, s.jt_keys, s.jt_rows, s.jt_mask, p->stream));
    p->stats.kernel_launches++;
    s.jt_generic = true;
    return BKGPU_OK;
}

// a two-table join child's own filter (Compiled::build_filter / probe_filter) over `nrows` rows of `cols` (every plan column, this child's at
// the rows' start) into *bits: "key not NULL and the conjunction TRUE".  `dropped`: matched[] of the build side, 2 where the conjunction is not TRUE
static int join_child_filter(bkgpu_plan* p, const Program& prog, int key_col, const DevCol* cols, int64_t nrows, uint8_t** bits, size_t* bits_cap, uint8_t* dropped) {
    const Compiled& c = p->c;
    int rc;
    if ((rc = ensure_buf(p, (void**)bits, bits_cap, ((size_t)nrows + 31) / 32 * 4 + 4))) return rc;
    StarFilter f; memset(&f, 0, sizeof f);
    for (size_t i = 0; i < c.cols.size(); i++) f.cols[i] = cols[i];
    f.prog = prog; f.key_col = key_col; f.nrows = nrows;
    CK(p, launch_star_dim_filter(f, (uint32_t*)*bits, dropped, p->stream));
    p->stats.kernel_launches++;
    return BKGPU_OK;
}

// the general probe's multimap (duplicate build keys, unmatched probe rows): built only when a batch needs it
static int join_generic_table(bkgpu_plan* p) {
    const Compiled& c = p->c;
    JoinState& j = p->join;
    JoinSide& s = j.side[0];
    if (s.jt_generic) return BKGPU_OK;
    int rc;
    DevCol key = store_col(s.store, (size_t)c.build_key_col);
    if (c.join_type != BK_INNER_JOIN) {   // one "found a partner" byte per build row
        if ((rc = ensure_buf(p, (void**)&j.matched, &j.matched_cap, (size_t)std::max<int64_t>(s.store.rows, 1)))) return rc;
        CK(p, cudaMemsetAsync(j.matched, 0, (size_t)std::max<int64_t>(s.store.rows, 1), p->stream));
        if (c.n_build_filter > 0) {   // (SEMI / ANTI) a row that fails its own filter is neither in the multimap nor in the tail
            const std::vector<DevCol> all = join_cols(p, nullptr);
            if ((rc = join_child_filter(p, c.build_filter, c.build_key_col, all.data(), s.store.rows, &s.keybits, &s.keybits_cap, j.matched))) return rc;
            key.validity = s.keybits;
        }
    }
    return join_build_multimap(p, s, key, c.join_key_prim);
}

// the probe child's own filter over one batch (`all`: every plan column): its bitmap becomes the probe key's validity for the batch, so a row that
// fails it finds no partner, as a row with a NULL key.  Never for FULL, where such a row would still come out NULL-extended.  A row that passes
// has a valid key: every row the aggregate or the sink sees reads the key column as before.
static int join_probe_filter(bkgpu_plan* p, std::vector<DevCol>& all, int64_t nrows) {
    const Compiled& c = p->c;
    JoinState& j = p->join;
    if (c.n_probe_filter == 0) return BKGPU_OK;
    const int rc = join_child_filter(p, c.probe_filter, c.probe_key_col, all.data(), nrows, &j.probe_bits, &j.probe_bits_cap, nullptr);
    all[(size_t)c.probe_key_col].validity = j.probe_bits;
    return rc;
}

static int join_probe_batch(bkgpu_plan* p, const DevCol* probe_cols, int64_t nrows, int64_t, bool) {
    const Compiled& c = p->c;
    JoinState& j = p->join;
    const JoinSide& s = j.side[0];
    std::vector<DevCol> all = join_cols(p, probe_cols);
    // ---- FK -> PK fast path: gather the build columns next to the probe rows, then the ordinary (lean) aggregate ----
    if (s.jf.mode != 0 && j.jp.mode != 0 && c.jfast && !p->force_generic && !j.no_fused_probe) {
        // ---- fused probe: the lean aggregate reads the foreign key and looks the group key up itself ----
        const Compiled& f = *c.jfast;
        std::vector<DevCol> fc(f.cols.size());
        const int key_fcol = f.direct_cols[(size_t)j.jp_key_pos];
        bool vec_ok = true;
        for (size_t i = 0; i < f.cols.size(); i++) {
            fc[i] = (int)i == key_fcol ? all[(size_t)c.probe_key_col] : all[(size_t)c.jfast_of_main[i]];
            if (((uintptr_t)fc[i].values & 31) != 0) vec_ok = false;
        }
        const int rc = launch_agg_batch(p, f, fc.data(), nrows, vec_ok, &j.jp);
        if (rc <= 0) return rc;   // launched (0) or failed (< 0); +1: this batch does not fit the lean kernel
    }
    if (s.jf.mode != 0 && c.jfast && !p->force_generic) {
        const Compiled& f = *c.jfast;
        const int64_t chunk = 16 << 20;   // the gathered chunk is re-read immediately: keep it L2-sized
        for (int64_t off = 0; off < nrows; off += chunk) {
            const int64_t n = std::min(chunk, nrows - off);
            GatherCols gc{}; std::vector<DevCol> fc(f.cols.size());
            int rc;
            for (size_t i = 0; i < f.cols.size(); i++) {
                const size_t m = (size_t)c.jfast_of_main[i];
                if (c.col_side[m] != 1) { fc[i] = col_at(all[m], off); continue; }
                if ((rc = store_reserve(p, j.chunk, m, chunk, chunk, false))) return rc;
                uint8_t* dst = j.chunk.cols[m].vals;
                gc.src[gc.n] = s.store.cols[m].vals; gc.dst[gc.n] = dst; gc.elem[gc.n] = storage_bytes(all[m].stype); gc.n++;
                fc[i] = all[m]; fc[i].values = dst; fc[i].validity = nullptr;
            }
            CK(p, cudaMemsetAsync(p->d_cursor + 1, 0, 4, p->stream));
            CK(p, launch_join_gather(col_at(all[(size_t)c.probe_key_col], off), c.cols[(size_t)c.probe_key_col].prim, c.join_key_prim, n, s.jf, gc, p->d_cursor + 1, p->stream));
            p->stats.kernel_launches++;
            uint32_t miss = 0;
            if ((rc = read_u32(p, p->d_cursor + 1, &miss))) return rc;
            if (miss) {   // some probe row has no partner (or a NULL key): this chunk takes the general probe
                std::vector<DevCol> sl(all);
                for (size_t i = 0; i < sl.size(); i++) if (c.col_side[i] == 0) sl[i] = col_at(all[i], off);
                if ((rc = join_generic_table(p))) return rc;
                if ((rc = launch_agg_batch(p, c, sl.data(), n, false))) return rc;
            } else {
                bool vec_ok = true;
                for (auto& d : fc) if (((uintptr_t)d.values & 31) != 0) vec_ok = false;
                if ((rc = launch_agg_batch(p, f, fc.data(), n, vec_ok))) return rc;
            }
        }
        return BKGPU_OK;
    }
    { int rc; if ((rc = join_generic_table(p)) || (rc = join_probe_filter(p, all, nrows))) return rc; }
    return launch_agg_batch(p, c, all.data(), nrows, false);
}

// the (probe row, build row) pairs of `n_probe` probe rows (`all`: every plan column, the probe side's at the rows' start), or of the
// outer-join tail, into j.pairs; *found = their number
static int join_pairs(bkgpu_plan* p, const std::vector<DevCol>& all, int64_t n_probe, bool tail, uint32_t* found) {
    const Compiled& c = p->c;
    JoinState& j = p->join;
    int rc;
    AggArgs a; memset(&a, 0, sizeof a);
    a.plan = c.ap; a.prog = c.prog; a.nrows = n_probe;
    const int ncols = (int)c.cols.size();
    for (int i = 0; i < ncols; i++) a.cols[i] = all[(size_t)i];
    a.n_cols = ncols;
    a.join = join_args(p, tail);
    if ((rc = ensure_buf(p, (void**)&j.cursor, &j.cursor_cap, 64))) return rc;
    *found = 0;
    return run_counted(p, (uint64_t)std::max<int64_t>(tail ? j.side[0].store.rows : n_probe, 1 << 12), j.cursor, found, [&](uint64_t want) -> int {
        if (want > 0x7FFFFFF0ull) return p->fail(BKGPU_ETOOBIG, "a probe batch joins to more than 2^31 rows: push smaller batches");
        int r;
        if ((r = ensure_buf(p, (void**)&j.pairs, &j.pairs_cap, (size_t)want * 8))) return r;
        CK(p, cudaMemsetAsync(j.cursor, 0, 4, p->stream));
        // (a rerun of a LEFT / FULL batch sets the same matched[] flags again: they only ever go from 0 to 1; a 2 is never in the multimap)
        CK(p, launch_join_pairs(a, j.pairs, (uint32_t)want, j.cursor, p->sm_count, p->stream));
        p->stats.kernel_launches++;
        return BKGPU_OK;
    });
}

// ---- a JOIN that returns rows (PK_JOIN): pairs -> gather -> the sink fragment (p->post_sort) ----
static int join_rows_emit(bkgpu_plan* p, const std::vector<DevCol>& all, int64_t n_probe, bool tail) {
    const Compiled& c = p->c;
    JoinState& j = p->join;
    int rc;
    uint32_t found = 0;
    rc = join_pairs(p, all, n_probe, tail, &found);
    if (rc || !found) return rc;
    const Compiled& pc = *c.post;
    const size_t nc = pc.cols.size();
    std::vector<DevCol> dc(std::max<size_t>(nc, 1));
    for (size_t k = 0; k < nc; k++) {   // sink column k = output column k = device column k of the join (plan.cpp::lower_join_rows)
        const RowStore::Col& d = p->post.cols[k];
        if ((rc = store_reserve(p, p->post, k, found, std::max<int64_t>((int64_t)found + found / 4, 1 << 16), true))) return rc;
        CK(p, launch_join_rows_gather(all[k], j.pairs, 2, c.col_side[k] == 1 ? 1 : 0, found, storage_bytes(prim_storage(d.prim)), d.vals, d.nulls, p->stream));
        if ((rc = store_pack(p, p->post, k, found, 16, nullptr, &dc[k]))) return rc;
    }
    p->stats.kernel_launches += 2 * (int64_t)nc;
    p->rows_passed_host += found;
    if ((rc = sort_push(p->post_sort, dc.data(), (int64_t)found, &p->stats))) return rc;
    CK(p, cudaStreamSynchronize(p->stream));   // the gather buffers are reused by the next batch
    return BKGPU_OK;
}
static int join_rows_batch(bkgpu_plan* p, const DevCol* probe_cols, int64_t nrows, int64_t, bool) {
    int rc;
    std::vector<DevCol> all = join_cols(p, probe_cols);
    if ((rc = join_generic_table(p)) || (rc = join_probe_filter(p, all, nrows))) return rc;
    return join_rows_emit(p, all, nrows, false);
}

// ---- FULL join under an aggregate (PK_JOIN_AGG): pairs -> gather -> the aggregate over the joined row (Compiled::jfast, whose predicate is
// the filter above the join).  Never the FK -> PK path: that assumes exactly one partner per probe row. ----
// the pairs of `n_probe` probe rows (or of the tail), every column jfast reads gathered from its pair (NULL on the side a pair lacks), the aggregate
static int full_join_agg(bkgpu_plan* p, const std::vector<DevCol>& all, int64_t n_probe, bool tail) {
    const Compiled& c = p->c;
    const Compiled& f = *c.jfast;
    JoinState& j = p->join;
    uint32_t found = 0;
    int rc = join_pairs(p, all, n_probe, tail, &found);
    if (rc || !found) return rc;
    std::vector<DevCol> fc(f.cols.size());
    for (size_t i = 0; i < f.cols.size(); i++) {
        const size_t m = (size_t)c.jfast_of_main[i];
        if ((rc = store_reserve(p, j.chunk, m, found, found, true))) return rc;
        const RowStore::Col& g = j.chunk.cols[m];
        CK(p, launch_join_rows_gather(all[m], j.pairs, 2, c.col_side[m] == 1 ? 1 : 0, found, storage_bytes(all[m].stype), g.vals, g.nulls, p->stream));
        DevCol packed;
        if ((rc = store_pack(p, j.chunk, m, found, 16, nullptr, &packed))) return rc;
        p->stats.kernel_launches += 2;
        fc[i] = all[m]; fc[i].values = g.vals; fc[i].validity = packed.validity;
    }
    return launch_agg_batch(p, f, fc.data(), found, true);
}
static int full_join_probe_batch(bkgpu_plan* p, const DevCol* probe_cols, int64_t nrows, int64_t, bool) {
    const Compiled& c = p->c;
    int rc;
    if ((rc = join_generic_table(p))) return rc;
    const std::vector<DevCol> all = join_cols(p, probe_cols);
    const int64_t chunk = 16 << 20;   // bounds the pairs and the gathered chunk
    for (int64_t off = 0; off < nrows; off += chunk) {
        std::vector<DevCol> sl(all);
        for (size_t i = 0; i < sl.size(); i++) if (c.col_side[i] == 0) sl[i] = col_at(all[i], off);
        if ((rc = full_join_agg(p, sl, std::min(chunk, nrows - off), false))) return rc;
    }
    return BKGPU_OK;
}

// LEFT / SEMI / ANTI_SEMI / FULL: once every probe batch has run, the preserved (build) side's rows the join type asks for go through the
// aggregate (PK_JOIN_AGG) or the sink (PK_JOIN) — unmatched rows NULL-extended (LEFT, FULL), matched rows (SEMI), unmatched rows (ANTI_SEMI);
// join_node.cpp:1200-1276
int join_tail(bkgpu_plan* p) {
    const Compiled& c = p->c;
    JoinState& j = p->join;
    if (c.join_type == BK_INNER_JOIN || j.side[0].store.rows == 0) return BKGPU_OK;
    int rc;
    if (!j.built && (rc = join_build_table(p))) return rc;
    if ((rc = join_generic_table(p))) return rc;
    const std::vector<DevCol> all = join_cols(p, nullptr);
    if (c.kind == PK_JOIN) return join_rows_emit(p, all, 0, true);
    if (c.join_type == BK_FULL_JOIN) return full_join_agg(p, all, 0, true);
    j.tail_launch = true;
    rc = launch_agg_batch(p, c, all.data(), j.side[0].store.rows, false);
    j.tail_launch = false;
    return rc;
}

// ---- star join (PK_STAR_AGG): every dimension is retained and indexed before the first fact batch ----
static int star_build(bkgpu_plan* p) {
    const Compiled& c = p->c;
    p->join.built = true;
    int rc;
    for (size_t d = 0; d < c.dims.size(); d++) {
        JoinSide& s = p->join.side[d];
        const StarDim& sd = c.dims[d];
        if ((rc = join_pack_validity(p, s))) return rc;
        s.jt_generic = false; s.jf = JoinFast{};
        if (s.store.rows == 0) continue;
        DevCol key = store_col(s.store, (size_t)sd.key_col);
        if (sd.n_filter > 0) {   // the build key's validity: the key is not NULL and the dimension's own conjuncts are TRUE
            if ((rc = ensure_buf(p, (void**)&s.keybits, &s.keybits_cap, ((size_t)s.store.rows + 31) / 32 * 4))) return rc;
            StarFilter f; memset(&f, 0, sizeof f);
            for (size_t i = 0; i < c.cols.size(); i++) if (c.col_side[i] == 1 + (int)d) f.cols[i] = store_col(s.store, i);
            f.prog = sd.filter; f.key_col = sd.key_col; f.nrows = s.store.rows;
            CK(p, launch_star_dim_filter(f, (uint32_t*)s.keybits, nullptr, p->stream));
            p->stats.kernel_launches++;
            key.validity = s.keybits;
        }
        // unique keys: the dense or packed index; duplicate keys (or 64-bit keys over a wide range): the multimap
        if ((rc = join_build_index(p, s, key, sd.cast_prim, false))) return rc;
        if (s.jf.mode == 0 && (rc = join_build_multimap(p, s, key, sd.cast_prim))) return rc;
    }
    return BKGPU_OK;
}

// the tuple buffer `k` with room for `n` tuples of `w` row ids
static int star_tuples(bkgpu_plan* p, int k, uint64_t n, int w) {
    if (n * (uint64_t)w > 0xFFFFFFF0ull) return p->fail(BKGPU_ETOOBIG, "a star join chunk joins to more than 2^32 row ids: push smaller batches");
    return ensure_buf(p, (void**)&p->join.tuples[k], &p->join.tuples_cap[k], (size_t)std::max<uint64_t>(n, 1) * (size_t)w * 4);
}

// A fact batch, chunk by chunk: k_star_probe keeps the rows with a partner in every dimension of unique keys, each dimension with duplicate
// keys expands the survivors (k_star_expand), the referenced columns are gathered side by side, and the aggregate runs over them as the
// virtual joined tuple (Compiled::jfast: the lean kernel when the shape fits).
static int star_probe_batch(bkgpu_plan* p, const DevCol* fact_cols, int64_t nrows, int64_t, bool vec_ok) {
    const Compiled& c = p->c;
    const Compiled& f = *c.jfast;
    JoinState& j = p->join;
    const int D = (int)c.dims.size(), W = 1 + D;
    for (int d = 0; d < D; d++) if (j.side[d].store.rows == 0) return BKGPU_OK;   // an empty dimension: no row joins
    const std::vector<DevCol> all = join_cols(p, fact_cols);
    int rc;
    const int64_t chunk = 16 << 20;
    for (int64_t off = 0; off < nrows; off += chunk) {
        const int64_t n = std::min(chunk, nrows - off);
        StarProbe sp; memset(&sp, 0, sizeof sp);
        sp.width = W; sp.nrows = n; sp.vec = vec_ok ? 1 : 0;
        for (int d = 0; d < D; d++) {
            if (j.side[d].jf.mode == 0) continue;
            const StarDim& sd = c.dims[(size_t)d];
            StarLookup& L = sp.d[sp.n++];
            L.fk = col_at(all[(size_t)sd.fk_col], off); L.from_prim = c.cols[(size_t)sd.fk_col].prim; L.cast_prim = sd.cast_prim; L.slot = 1 + d; L.jf = j.side[d].jf;
        }
        if ((rc = star_tuples(p, 0, (uint64_t)n, W))) return rc;
        CK(p, launch_star_probe(sp, j.tuples[0], p->d_cursor + 1, p->sm_count, p->stream));
        p->stats.kernel_launches++;
        uint32_t found = 0;
        if ((rc = read_u32(p, p->d_cursor + 1, &found))) return rc;
        int cur = 0;
        for (int d = 0; d < D && found; d++) {   // dimensions with duplicate keys: one expansion pass each
            const JoinSide& s = j.side[d];
            if (s.jf.mode != 0) continue;
            const StarDim& sd = c.dims[(size_t)d];
            const DevCol fk = col_at(all[(size_t)sd.fk_col], off);
            uint32_t got = 0;
            rc = run_counted(p, j.star_expand_cap > 0 ? (uint64_t)j.star_expand_cap : std::max<uint64_t>(2 * (uint64_t)found, 4096), p->d_cursor + 1, &got,
                             [&](uint64_t cap) -> int {
                int r;
                if ((r = star_tuples(p, 1 - cur, cap, W))) return r;
                CK(p, launch_star_expand(fk, c.cols[(size_t)sd.fk_col].prim, sd.cast_prim, s.jt_keys, s.jt_rows, s.jt_mask, j.tuples[cur], found,
                                         W, 1 + d, j.tuples[1 - cur], (uint32_t)cap, p->d_cursor + 1, p->stream));
                p->stats.kernel_launches++;
                return BKGPU_OK;
            });
            if (rc) return rc;
            found = got; cur = 1 - cur;
        }
        if (!found) continue;
        // the joined chunk: every column the aggregate reads, gathered from its tuple's row
        std::vector<DevCol> fc(f.cols.size());
        for (size_t i = 0; i < f.cols.size(); i++) {
            const size_t m = (size_t)c.jfast_of_main[i];
            const int side = c.col_side[m];
            const DevCol src = side == 0 ? col_at(all[m], off) : all[m];
            if ((rc = store_reserve(p, j.chunk, m, found, found, src.validity != nullptr))) return rc;   // NULLs travel along: null bytes, then a bitmap
            const RowStore::Col& g = j.chunk.cols[m];
            fc[i] = src; fc[i].values = g.vals; fc[i].validity = nullptr;
            CK(p, launch_join_rows_gather(src, j.tuples[cur], W, side, found, storage_bytes(src.stype), g.vals, src.validity ? g.nulls : nullptr, p->stream));
            p->stats.kernel_launches++;
            if (src.validity) {
                DevCol packed;
                if ((rc = store_pack(p, j.chunk, m, found, 16, nullptr, &packed))) return rc;
                p->stats.kernel_launches++;
                fc[i].validity = packed.validity;
            }
        }
        if ((rc = launch_agg_batch(p, f, fc.data(), found, true))) return rc;
    }
    return BKGPU_OK;
}

// a batch of a build table — the two-table join's build side, a star join's dimensions — is retained; any other batch is probed
int join_push(bkgpu_plan* p, const bkgpu_column* cols, int ncols, int64_t nrows, int on_device) {
    const Compiled& c = p->c;
    JoinState& j = p->join;
    const bool star = c.kind == PK_STAR_AGG;
    if (j.chunk.cols.empty()) {   // the stores' columns, by plan column: a build side holds its own table's
        store_init(j.chunk, c.cols);
        for (int d = 0; d < 4; d++) {
            store_init(j.side[d].store, c.cols);
            for (size_t i = 0; i < c.cols.size(); i++) if (c.col_side[i] != 1 + d) j.side[d].store.cols[i].prim = -1;
        }
    }
    int side = 0;   // (the Compiled::col_side value of the build table's columns)
    if (!star) { for (int k = 0; k < ncols; k++) if (cols[k].tuple_id == c.build_tuple) side = 1; }
    else for (size_t d = 0; d < c.dims.size() && !side; d++) for (int k = 0; k < ncols; k++) if (cols[k].tuple_id == c.dims[d].tuple_id) side = 1 + (int)d;
    if (side) return join_retain_build(p, side, cols, ncols, nrows, on_device);
    if (!j.built) { int rc = star ? star_build(p) : join_build_table(p); if (rc) return rc; }
    if (j.probe_want.empty()) for (size_t i = 0; i < c.cols.size(); i++) if (c.col_side[i] == 0) { j.probe_want.push_back(c.cols[i]); j.probe_map.push_back((int)i); }
    return feed(p, j.probe_want, cols, ncols, nrows, on_device, star ? star_probe_batch : c.kind == PK_JOIN ? join_rows_batch :
                                                                c.join_type == BK_FULL_JOIN ? full_join_probe_batch : join_probe_batch);
}

void join_reset(bkgpu_plan* p) {
    p->join.built = false;
    for (JoinSide& s : p->join.side) {
        s.store.rows = 0; s.jt_generic = false;
        for (RowStore::Col& col : s.store.cols) col.nullable = false;   // (the previous run's bitmaps are not read again)
    }
}
