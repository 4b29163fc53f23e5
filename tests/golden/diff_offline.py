"""The checker of the offline merge -- oracle/offline.py's restatement -- against the REAL LocalFeatureMerger.merge
(retrieval/base.py:412-468, local_merger.py:29-104) on 300 random workloads (tests/golden/gen_offline.merge_inputs: int64,
int32, string and int32-pair keys, as-of and exact-key joins, 1 to 3 feature sets, s / ms / us / ns units and cross-unit
casts, colliding column names, unknown keys, entity rows before every feature row).  Frames, drop columns, the resulting
timestamp column and exceptions compared.

    python -m tests.golden.diff_offline     # needs the reference sources importable (tests/golden/_refshim.py)
"""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
import pandas as pd  # noqa: E402

from oracle import offline as oo  # noqa: E402
from tests.golden import gen_offline  # noqa: E402


def main(n=300):
    from tests.golden import _refshim

    _refshim.install()
    import logging

    logging.disable(logging.INFO)
    for seed in range(1000, 1000 + n):
        want = gen_offline.run_merge(gen_offline.reference_merge, seed)
        got = gen_offline.run_merge(oo.merge, seed)
        if isinstance(want, dict) or isinstance(got, dict):
            same = want == got if isinstance(want, dict) and isinstance(got, dict) else False
        else:
            try:
                pd.testing.assert_frame_equal(got[0], want[0], check_exact=True)
                same = got[1:] == want[1:]
            except AssertionError:
                same = False
        if not same:
            print("DIFF at seed", seed)
            print("  ref :", want if isinstance(want, dict) else (want[0].head(), want[1:]))
            print("  mine:", got if isinstance(got, dict) else (got[0].head(), got[1:]))
            return 1
    print("identical on", n, "random offline merges")
    return 0


if __name__ == "__main__":
    sys.exit(main())
