"""The wgmma exact scan's conservative filter (usearch_b200/csrc/exact_i8.h) never rejects a column that belongs in the
k-best list, natively: tests/native/test_exact_i8_filter.cpp over 10^7 random (ab, a2, b2) triples and the adversarial
families (cos ties near distance 1, clamped duplicates, zero norms, sums past 2^24), ip / l2sq / cos in both operand
orders, with the distances held bit-equal to the pinned reference metrics."""
import os
import subprocess

import common


def test_exact_i8_filter_passes_every_column_inside_the_worst(tmp_path):
    exe = str(tmp_path / "test_exact_i8_filter")
    subprocess.run(["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-Wall", "-Wextra", "-Werror",
                    "-I", os.path.join(common.ROOT, "oracle"), "-I", os.path.join(common.ROOT, "usearch_b200", "csrc"),
                    os.path.join(common.ROOT, "tests", "native", "test_exact_i8_filter.cpp"), "-o", exe, "-lm"], check=True)
    out = subprocess.run([exe], capture_output=True, text=True)
    assert out.returncode == 0, out.stdout[-4000:] + out.stderr
    assert "failures: 0" in out.stdout
