// window.h — K6: the window stage (WINDOW -> SORT pairs, plan kind PK_WINDOW) over the rows a SortState retained.
#pragma once
#include <stdint.h>
#include <vector>
#include "../include/bkgpu.h"
#include "sort.h"

namespace bk {

// Runs every stage of p->c.win over the rows p->sort retained (stable radix sort when a stage's keys change, then the window functions),
// and writes the output rows (the scan tuple's slots, then one column per window function) into p->result in the top stage's order after
// LIMIT / OFFSET, or — when p->post is set (the query's ORDER BY, c.post) — in the post fragment's order.  p->stats.main_kernel_* report
// the window kernels (sorts excluded).
int window_finish(bkgpu_plan* p);

}  // namespace bk
