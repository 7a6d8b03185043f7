// window.h — K6: the window stage (WINDOW -> SORT pairs, plan kind PK_WINDOW) over the rows a SortState retained.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <string>
#include <vector>
#include "../include/bkgpu.h"
#include "plan.h"
#include "sort.h"

namespace bk {

// Runs every stage of c.win over the rows `rows` retained (stable radix sort when a stage's keys change, then the window functions), and
// returns the output rows (the scan tuple's slots, then one column per window function) in the top stage's order after LIMIT / OFFSET,
// or — when `post` is given (the query's ORDER BY, c.post) — in the post fragment's order.  stats->main_kernel_* report the window
// kernels (sorts excluded).
int window_finish(const Compiled& c, SortState* rows, SortState* post, cudaStream_t stream, bkgpu_stats* stats,
                  std::vector<SortOutCol>& out, int64_t* nrows, std::string& err);

}  // namespace bk
