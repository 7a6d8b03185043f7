// window.h — K6: the window stage (WINDOW -> SORT pairs, plan kind PK_WINDOW) over the rows a SortState retained.
#pragma once
#include <stdint.h>
#include <vector>
#include "../include/bkgpu.h"
#include "sort.h"

namespace bk {

// Runs every stage of w.win (a PK_WINDOW fragment: the plan itself over a scan, or the post fragment above an aggregate) over the rows
// `rows` retained (stable radix sort when a stage's keys change, then the window functions), and writes the output rows (w's input
// columns, then one column per window function) into p->result in the top stage's order after LIMIT / OFFSET, or — when `outer` is set
// (the query's ORDER BY, w.post) — in that fragment's order.  stats->main_kernel_* report the window kernels (sorts excluded).
int window_finish(bkgpu_plan* p, const Compiled& w, SortState* rows, SortState* outer, bkgpu_stats* stats);

}  // namespace bk
