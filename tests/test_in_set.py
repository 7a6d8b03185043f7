"""CPU: the hashed IN set (csrc/in_set.h) against a linear scan with OP_IN's comparison, through the driver tests/cpp/in_set_check.cpp —
every value class, lists of 1 to 10^6 entries with duplicates and with every entry equal, members, their neighbours and random probes,
the integer extremes, ±0.0, NaN, ±inf and denormals, and the table's empty-slot sentinel as a member and as a probe."""
import os
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_set_lookup_equals_a_linear_scan(tmp_path):
    exe = str(tmp_path / "in_set_check")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-Wall", "-Wextra", "-Werror", "-I", os.path.join(ROOT, "csrc"),
                           os.path.join(ROOT, "tests", "cpp", "in_set_check.cpp"), "-o", exe])
    out = subprocess.run([exe], capture_output=True, text=True, timeout=600)
    assert out.returncode == 0 and "in_set_check ok" in out.stdout, out.stdout[-3000:]
