"""The numpy restatement of the online table's hash (tests/table_hash.py) against csrc/b2s_hash.cuh itself, and the
key-crafting helper the enrichment path tests build their probe chains with.  CPU only."""

import os
import shutil
import subprocess

import numpy as np
import pytest

from tests import table_hash as th

HASH_HEADER = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "mlrun_b200", "csrc", "b2s_hash.cuh")
I64_MIN, I64_MAX = np.iinfo(np.int64).min, np.iinfo(np.int64).max
DRIVER = r"""
#include <cstdio>
#include "b2s_hash.cuh"
int main() {
  long long k;
  while (std::scanf("%lld", &k) == 1) std::printf("%llu\n", (unsigned long long)b2s::mix64((uint64_t)k));
  return 0;
}
"""


def seeded_keys(n=10000, seed=1):
    rng = np.random.default_rng(seed)
    edge = np.array([0, 1, -1, I64_MIN, I64_MAX, I64_MIN + 1, I64_MAX - 1, 1 << 32, -(1 << 32)], dtype=np.int64)
    return np.concatenate([edge, rng.integers(I64_MIN, I64_MAX, size=n - len(edge), dtype=np.int64, endpoint=True)])


def test_mix64_matches_the_header(tmp_path):
    """a host build of the header's own mix64 (the kernels' hash) prints the same words as the numpy restatement"""
    cxx = shutil.which("g++") or shutil.which("c++")
    if cxx is None:
        pytest.skip("no host C++ compiler")
    src = tmp_path / "mix.cpp"
    src.write_text(DRIVER)
    exe = tmp_path / "mix"
    subprocess.run([cxx, "-O1", "-std=c++17", "-D__host__=", "-D__device__=", f"-I{os.path.dirname(HASH_HEADER)}",
                    str(src), "-o", str(exe)], check=True)
    keys = seeded_keys()
    out = subprocess.run([str(exe)], input="\n".join(str(k) for k in keys.tolist()), capture_output=True, text=True,
                         check=True).stdout.split()
    assert len(out) == len(keys)
    np.testing.assert_array_equal(np.array([int(w) for w in out], dtype=np.uint64), th.mix64(keys))
    assert th.mix64(np.array([0]))[0] == 0  # key 0 homes at slot 0, where an empty slot also holds key 0


def test_unmix64_inverts_mix64():
    keys = seeded_keys(seed=2)
    np.testing.assert_array_equal(th.unmix64(th.mix64(keys)), keys)
    words = seeded_keys(seed=3).view(np.uint64)
    np.testing.assert_array_equal(th.mix64(th.unmix64(words)), words)


def test_capacity_rule():
    assert [th.capacity(n) for n in (1, 8, 9, 16, 17, 1024, 1025)] == [16, 16, 32, 32, 64, 2048, 4096]


@pytest.mark.parametrize("cap", [16, 1024, 1 << 21])
def test_keys_with_home_slots(cap):
    rng = np.random.default_rng(cap)
    slots = np.concatenate([np.full(50, cap - 3), rng.integers(0, cap, size=200), [0, cap - 1]])
    keys = th.keys_with_home_slots(slots, cap, rng)
    assert keys.dtype == np.int64 and len(set(keys.tolist())) == len(keys)
    np.testing.assert_array_equal(th.home_slot(keys, cap), slots)
    more = th.keys_with_home_slots(slots[:60], cap, rng, exclude=keys)
    assert not set(more.tolist()) & set(keys.tolist())
    np.testing.assert_array_equal(th.home_slot(more, cap), slots[:60])


def test_probe_layout_wraps():
    """keys all homed at cap - 3 fill cap - 3, cap - 2, cap - 1, 0, 1, ...: the chain wraps past the last slot"""
    cap = th.capacity(8)
    keys = th.keys_with_home_slots(np.full(8, cap - 3), cap, np.random.default_rng(0))
    layout = th.probe_layout(keys, cap)
    assert sorted(layout) == [0, 1, 2, 3, 4, cap - 3, cap - 2, cap - 1]
    assert layout[cap - 3] == keys[0] and layout[4] == keys[7]
