"""The search kernel evaluates the cos / ip f32 prefilter bound with its query-only terms computed once per query
(prefilter_bound.h, pf_query_bound). That form must return the same bits as the per-candidate one, natively:
tests/native/test_prefilter_bound_hoisted.cpp over 10^7 random and the adversarial pairs."""
import os
import subprocess

import common


def test_per_query_bound_returns_the_same_bits(tmp_path):
    exe = str(tmp_path / "test_prefilter_bound_hoisted")
    subprocess.run(["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-Wall", "-Wextra", "-Werror",
                    "-I", os.path.join(common.ROOT, "oracle"), "-I", os.path.join(common.ROOT, "usearch_b200", "csrc"),
                    os.path.join(common.ROOT, "tests", "native", "test_prefilter_bound_hoisted.cpp"), "-o", exe, "-lm"],
                   check=True)
    out = subprocess.run([exe], capture_output=True, text=True)
    assert out.returncode == 0, out.stdout + out.stderr
    assert "failures: 0" in out.stdout
