"""The context's memory owner (csrc/ctx_memory.h), compiled with g++ against fake CUDA allocation calls
(tests/hostcheck/ctx_memory_host.cpp): the grow rule, the drain before a free, zero-fill, retry after a failed
allocation, freeing on destruction, and the scratch layout's alignment, order and two passes."""
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CUDA_INC = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "include")
CASES = ["no_call_when_big_enough", "drains_before_it_frees", "zero_fill_covers_the_new_allocation",
         "failed_allocation_leaves_it_empty", "destroying_the_owner_frees_everything",
         "layout_is_aligned_ordered_and_sized_once"]


@pytest.fixture(scope="module")
def exe(tmp_path_factory):
    out = os.path.join(str(tmp_path_factory.mktemp("ctx_memory")), "ctx_memory_host")
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-Wall", "-Wno-attributes", "-I" + CUDA_INC, "-o", out,
                           os.path.join(ROOT, "tests", "hostcheck", "ctx_memory_host.cpp")])
    return out


@pytest.mark.parametrize("case", CASES)
def test_ctx_memory_on_host(exe, case):
    r = subprocess.run([exe, case], capture_output=True, text=True)
    assert r.returncode == 0 and r.stdout.strip() == "ok", r.stdout + r.stderr
