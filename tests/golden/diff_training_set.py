"""The checker of training sets -- tests/training_oracle.py's restatement of the spine, the label append and `*` exclusion,
dropna and float64 columns -- against the REAL BaseMerger.start on the local engine (tests/golden/gen_training_set.py) on
300 random workloads.  Frames (values, dtypes, column order, row labels) and exceptions compared.

    python -m tests.golden.diff_training_set     # needs the reference sources importable (tests/golden/_refshim.py)
"""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
import pandas as pd  # noqa: E402

from tests.golden import gen_training_set as gen  # noqa: E402


def oracle_training_set(frames, features, label_feature, entity_rows, entity_timestamp_column, with_indexes):
    from tests import training_oracle

    return training_oracle.get_offline_features(frames, features, entity_rows, entity_timestamp_column, with_indexes=with_indexes,
                                   label_feature=label_feature)


def same(got, want):
    """the oracle's outcome against the reference's: its error message (the oracle raises ValueError for the reference's
    MLRunInvalidArgumentError), or an identical frame"""
    if isinstance(want, dict) or isinstance(got, dict):
        return isinstance(want, dict) and isinstance(got, dict) and got["message"] == want["message"]
    try:
        pd.testing.assert_frame_equal(got, want, check_exact=True)
        return True
    except AssertionError:
        return False


def main(n=300):
    from tests.golden import _refshim

    _refshim.install()
    import logging

    logging.disable(logging.WARNING)
    for seed in range(1000, 1000 + n):
        want = gen.run(gen.reference_training_set, seed)
        got = gen.run(oracle_training_set, seed)
        if not same(got, want):
            print("DIFF at seed", seed)
            print("  ref :", want)
            print("  mine:", got)
            return 1
    print("identical on", n, "random training sets")
    return 0


if __name__ == "__main__":
    sys.exit(main())
