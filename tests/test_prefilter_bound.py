"""The int8-shadow lower bound of the cos / ip f32 prefilter (usearch_b200/csrc/prefilter_bound.h) against the pinned
reference metrics, natively: tests/native/test_prefilter_bound.cpp over 10^7 random and the adversarial pairs."""
import os
import subprocess

import common


def test_prefilter_bound_never_exceeds_the_pinned_distance(tmp_path):
    exe = str(tmp_path / "test_prefilter_bound")
    subprocess.run(["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-Wall", "-Wextra", "-Werror",
                    "-I", os.path.join(common.ROOT, "oracle"), "-I", os.path.join(common.ROOT, "usearch_b200", "csrc"),
                    os.path.join(common.ROOT, "tests", "native", "test_prefilter_bound.cpp"), "-o", exe, "-lm"], check=True)
    out = subprocess.run([exe], capture_output=True, text=True)
    assert out.returncode == 0, out.stdout + out.stderr
    assert "failures: 0" in out.stdout
