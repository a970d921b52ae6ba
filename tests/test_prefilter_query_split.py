"""The int8 split of the query that the cos / ip f32 prefilter multiplies on the tensor cores, and the lower bound it
feeds (usearch_b200/csrc/prefilter_bound.h), against the pinned reference metrics, natively:
tests/native/test_prefilter_query_split.cpp over 10^7 random pairs, the adversarial pairs and queries made for the
split."""
import os
import subprocess

import common


def test_prefilter_query_split_bound_never_exceeds_the_pinned_distance(tmp_path):
    exe = str(tmp_path / "test_prefilter_query_split")
    subprocess.run(["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-Wall", "-Wextra", "-Werror",
                    "-I", os.path.join(common.ROOT, "oracle"), "-I", os.path.join(common.ROOT, "usearch_b200", "csrc"),
                    os.path.join(common.ROOT, "tests", "native", "test_prefilter_query_split.cpp"), "-o", exe, "-lm"],
                   check=True)
    out = subprocess.run([exe], capture_output=True, text=True)
    assert out.returncode == 0, out.stdout + out.stderr
    assert "failures: 0" in out.stdout
