// The C++ row <-> column bridge (host/bkgpu_host.hpp's Chunk) with HLL sketches: rows holding 16400-byte RAW sketches become a column
// batch and come back as the same bytes; a sketch of another length is refused.  No GPU: only the bridge runs.
//   g++ -std=c++17 -I include -I host tests/cpp/hll_chunk_check.cpp -L baikaldb_b200 -l:libbkgpu.so && ./a.out
// Prints "ok rows=N" and exits 0, or names the first mismatch and exits 1.
#include <stdio.h>
#include "bkgpu_host.hpp"

int main() {
    using bkgpu::Chunk; using bkgpu::Value; using bkgpu::MemRowValues;
    Chunk ch({{0, 1, BK_INT32}, {9, 1, BK_HLL}});
    std::vector<MemRowValues> rows;
    for (int r = 0; r < 21; r++) {
        std::string sk(16400, '\0');
        memcpy(&sk[0], "HYLL", 4); sk[4] = (char)255;
        if (r % 2) sk[15] = (char)0x80;
        for (int i = 0; i < 16384; i += 97) sk[16 + i] = (char)((r * 7 + i) % 52);
        MemRowValues row{Value::of_int(r), r % 5 == 3 ? Value() : Value::of_bytes(sk)};
        if (ch.add_row(row)) { printf("add_row failed at %d\n", r); return 1; }
        rows.push_back(row);
    }
    if (ch.add_row({Value::of_int(99), Value::of_bytes(std::string(16, 'x'))}) != -1) { printf("a short sketch was accepted\n"); return 1; }
    bkgpu::RowBatch b = ch.finish();
    if (b.columns[1].elem_size != 16400 || b.columns[1].values.size() != (size_t)21 * 16400) { printf("column layout\n"); return 1; }
    std::vector<MemRowValues> back = Chunk::to_rows(b);
    if (back.size() != rows.size()) { printf("row count %zu\n", back.size()); return 1; }
    for (size_t r = 0; r < rows.size(); r++) {
        if (back[r][0].i64 != rows[r][0].i64 || back[r][1].is_null != rows[r][1].is_null || back[r][1].bytes != rows[r][1].bytes) {
            printf("row %zu differs\n", r); return 1;
        }
    }
    printf("ok rows=%zu\n", back.size());
    return 0;
}
