// rb_host_check.cpp — tests/test_rb_plan.py: the C++ host mirror refuses, when it is initialised, a plan whose result holds rb_build_agg's
// BITMAP column, and says why when opened; another plan initialises.  stdin: repeated { uint32 bytes; plan bytes }.  Needs no GPU.
#include <stdint.h>
#include <stdio.h>
#include <vector>
#include "bkgpu_host.hpp"

int main() {
    uint32_t n;
    while (fread(&n, 4, 1, stdin) == 1) {
        std::vector<uint8_t> plan(n);
        if (fread(plan.data(), 1, n, stdin) != n) return 2;
        bkgpu::GpuExecNode node;
        const int rc = node.init_serialized(plan);
        if (rc == 0) { printf("rc=0\n"); continue; }
        bkgpu::RuntimeState st;
        if (node.open(&st) != -1 || st.error_code != rc) return 3;
        printf("rc=%d %s\n", rc, st.error_msg.c_str());
    }
    return 0;
}
