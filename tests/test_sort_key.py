"""CPU: the sort key image (csrc/sort_key.h, shared by top-k, the radix sort, the multi-GPU merge and the window stage) against
ExprValue::compare, through the driver tests/cpp/sort_key_check.cpp — INT64 / UINT64 / DOUBLE images, ascending and descending, over all
pairs of the type extremes, ±0.0 (equal keys, as in MemRowCompare), ±denormals, ±DBL_MIN, ±DBL_MAX, ±Inf and 10^5 random pairs per class;
where NaN lands is pinned separately."""
import os
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_image_order_equals_expr_value_compare(tmp_path):
    exe = str(tmp_path / "sort_key_check")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-Wall", "-Wextra", "-Werror", "-I", os.path.join(ROOT, "csrc"),
                           os.path.join(ROOT, "tests", "cpp", "sort_key_check.cpp"), "-o", exe])
    out = subprocess.run([exe], capture_output=True, text=True, timeout=600)
    assert out.returncode == 0 and "sort_key_check ok" in out.stdout, out.stdout[-3000:]
