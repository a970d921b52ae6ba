"""The search's NaN rules for `next` and `top` (usearch_b200/csrc/search_order.h) against std::lower_bound and a
restatement of max_heap_gt, natively: tests/native/test_search_order_rules.cpp over random push / pop / insert
sequences drawn from NaN, +-inf, +-0, ties and finite values."""
import os
import re
import subprocess

import common


def test_heap_pop_and_top_position_follow_the_reference(tmp_path):
    exe = str(tmp_path / "test_search_order_rules")
    subprocess.run(["g++", "-std=c++17", "-O2", "-Wall", "-Wextra", "-Werror",
                    "-I", os.path.join(common.ROOT, "usearch_b200", "csrc"),
                    os.path.join(common.ROOT, "tests", "native", "test_search_order_rules.cpp"), "-o", exe], check=True)
    out = subprocess.run([exe, "100000"], capture_output=True, text=True)
    assert out.returncode == 0, out.stdout + out.stderr
    m = re.search(r"pops: (\d+) \(NaN entries seen (\d+)\), top inserts: (\d+) \(probed (\d+)\), failures: 0", out.stdout)
    assert m, out.stdout
    pops, nan_entries, inserts, probed = map(int, m.groups())
    assert pops > 10**6 and nan_entries > 10**5, out.stdout  # the pops met NaN heaps
    assert inserts > 10**5 and probed > 10**5, out.stdout  # and `top` was probed behind a NaN
