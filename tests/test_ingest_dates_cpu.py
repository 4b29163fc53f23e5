"""DateExtractor arithmetic of the columnar ingest kernel (csrc/b2s_dates.cuh: floor_div, civil_from_days, date_part),
compiled for the host and compared with pandas over every day datetime64[ns] holds.  CPU only."""

import os
import shutil
import subprocess

import numpy as np
import pytest

from tests import ingest_dates as idt

CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "mlrun_b200", "csrc")
DRIVER = r"""
#include <cstdio>
#include <vector>
#include "b2s_dates.cuh"
int main(int argc, char** argv) {
  std::FILE* in = std::fopen(argv[1], "rb");
  std::vector<long long> ts;
  long long v;
  while (std::fread(&v, sizeof v, 1, in) == 1) ts.push_back(v);
  std::fclose(in);
  std::vector<int> out(ts.size() * (b2s::DP_LAST + 1));
  for (size_t i = 0; i < ts.size(); ++i)
    for (int p = 0; p <= b2s::DP_LAST; ++p) out[p * ts.size() + i] = b2s::date_part(ts[i], p);
  std::FILE* o = std::fopen(argv[2], "wb");
  std::fwrite(out.data(), sizeof(int), out.size(), o);
  return std::fclose(o);
}
"""


@pytest.fixture(scope="module")
def host_parts(tmp_path_factory):
    """{part: int32 array} from a host build of the header's own date_part over idt.exhaustive_timestamps()"""
    cxx = shutil.which("g++") or shutil.which("c++")
    if cxx is None:
        pytest.skip("no host C++ compiler")
    d = tmp_path_factory.mktemp("dates")
    (d / "dates.cpp").write_text(DRIVER)
    exe = d / "dates"
    subprocess.run([cxx, "-O2", "-std=c++17", "-D__device__=", "-D__forceinline__=inline", "-D__noinline__=", f"-I{CSRC}",
                    str(d / "dates.cpp"), "-o", str(exe)], check=True)
    ts = idt.exhaustive_timestamps()
    ts.tofile(d / "ts.bin")
    subprocess.run([str(exe), str(d / "ts.bin"), str(d / "parts.bin")], check=True)
    parts = np.fromfile(d / "parts.bin", dtype=np.int32).reshape(len(idt.PARTS), len(ts))
    return ts, parts


def test_the_set_reaches_every_edge():
    ts = idt.exhaustive_timestamps()
    assert len(ts) > 1_700_000 and len(np.unique(ts)) == len(ts)
    assert ts.min() == idt.I64_MIN + 1 and ts.max() == idt.I64_MAX
    assert np.isin([-1, -idt.NS_S, -idt.NS_S - 1, -idt.NS_S + 1], ts).all()
    years = idt.pandas_part(ts, 0)
    assert years.min() == 1677 and years.max() == 2262


@pytest.mark.parametrize("part", sorted(idt.PARTS), ids=lambda p: idt.PARTS[p])
def test_date_part_matches_pandas(host_parts, part):
    ts, parts = host_parts
    want = idt.pandas_part(ts, part)
    got = parts[part].astype(np.int64)
    bad = np.flatnonzero(got != want)
    assert bad.size == 0, (f"{bad.size} differences, first at {ts[bad[0]].view('datetime64[ns]')}: "
                           f"{got[bad[0]]} != {want[bad[0]]}")


def test_sub_second_instants_before_the_epoch(host_parts):
    """-1 ns is 1969-12-31 23:59:59 (floor division, not truncation)"""
    ts, parts = host_parts
    i = int(np.flatnonzero(ts == -1)[0])
    assert [int(parts[p][i]) for p in range(6)] == [1969, 12, 31, 23, 59, 59]
