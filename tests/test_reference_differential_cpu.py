"""The kernels' three CHECKERS -- the batched scoring oracle, the columnar ingest oracle, the enrichment oracle -- against what
the REAL reference classes returned on seeded random workloads.  The reference's outputs are stored under tests/golden/
(ref_hot_path.json.xz, ref_ingest.npz, ref_online.json.xz; `python -m tests.golden.<script> --record` writes them where the
reference sources are importable), so the comparison runs on every machine.  Each check runs in its own process, as the live
scripts do.  The other differential scripts (`python -m tests.golden.run_diffs`, ~3 minutes, live only) stay out of the suite."""
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.parametrize("script,verdict", [("diff_hot_path", "the batched oracle equals the real reference"),
                                            ("diff_ingest", "ingest_columns equals the real reference"),
                                            ("diff_online", "identical on 500 random online services")])
def test_kernel_checkers_equal_the_real_reference(script, verdict):
    done = subprocess.run([sys.executable, "-m", f"tests.golden.{script}", "--golden"], cwd=ROOT, capture_output=True, text=True,
                          timeout=600)
    assert done.returncode == 0, (done.stdout[-1500:], done.stderr[-1500:])
    assert verdict in done.stdout, done.stdout[-800:]
