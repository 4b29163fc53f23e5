"""The checker of `columns_kernel` -- oracle/ingest.py `ingest_columns`, the vectorised restatement of the feature-set ingest
graph -- against the REAL reference step classes walking the frame one row at a time (storey-engine semantics: DataframeSource
emits a dict per row, every row goes through the steps' `_do_storey`, ReduceToDataFrame re-assembles; ingestion.py:38-127),
build container only: random config-5-shaped workloads (float32 columns with NaN, categorical codes with out-of-vocabulary
values, counters, a timestamp; Imputer -> MapValues(ranges, with originals) -> OneHotEncoder -> DateExtractor -> DropFeatures ->
FeaturesetValidator) at several widths and seeds.  Frames compared exactly (values, column order), violations by count.

    python -m tests.golden.diff_ingest             # live, needs the reference sources importable (tests/golden/_refshim.py)
    python -m tests.golden.diff_ingest --record    # live, and store the reference's frames in ref_ingest.npz
    python -m tests.golden.diff_ingest --golden    # against the stored frames: runs anywhere
"""
import contextlib
import io
import os
import random
import sys
import types

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
import numpy as np  # noqa: E402
import pandas as pd  # noqa: E402

from mlrun_b200.synthetic import ingest_workload  # noqa: E402
from oracle import ingest as oingest  # noqa: E402
from oracle import transforms as otransforms  # noqa: E402


class RefSteps:
    """the `api` object IngestWorkload.build_steps wants, over the real classes"""

    def __init__(self, ref):
        self.ref = ref
        self.Imputer, self.MapValues, self.OneHotEncoder = ref.Imputer, ref.MapValues, ref.OneHotEncoder
        self.DateExtractor, self.DropFeatures = ref.DateExtractor, ref.DropFeatures

    @staticmethod
    def MinMaxValidator(**kw):
        return kw

    def FeaturesetValidator(self, validators):
        return self.ref.validator_step(validators, None)


def reference_rows(steps, df):
    out, printed = [], io.StringIO()
    with contextlib.redirect_stdout(printed):
        for row in df.to_dict("records"):
            body = row
            for step in steps:
                if type(step).__name__ == "FeaturesetValidator":
                    step.do(types.SimpleNamespace(body=body, key=None))
                else:
                    body = step.do(body)
            out.append(body)
    return pd.DataFrame(out, index=df.index), len([ln for ln in printed.getvalue().splitlines() if ln.strip()])


GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "ref_ingest.npz")


def cases():
    """the 12 seeded workloads, in order"""
    rnd = random.Random(41)
    for case in range(12):
        yield case, ingest_workload(n_rows=rnd.randint(150, 400), seed=300 + case, n_f32=rnd.choice([24, 32, 48]), n_cat=rnd.choice([8, 12]),
                                    n_counter=rnd.choice([2, 5]), nan_frac=rnd.choice([0.02, 0.1, 0.3]))


def reference_outputs():
    """per case: the reference's frame as {column: values} (column order kept) and the number of violations it printed"""
    from tests.golden import api_reference as ref

    steps_api = RefSteps(ref)
    outs = []
    for _case, wl in cases():
        want, n_printed = reference_rows(wl.build_steps(steps_api), wl.df)
        outs.append(({c: want[c].to_numpy() for c in want.columns}, n_printed))
    return outs


def check(want_all):
    rows = 0
    for (case, wl), (want, n_printed) in zip(cases(), want_all, strict=True):
        with contextlib.redirect_stdout(io.StringIO()):
            got, violations = oingest.ingest_columns(wl.build_steps(otransforms), wl.df)
        assert list(got.columns) == list(want), (case, list(got.columns)[:8], list(want)[:8])
        for c, b in want.items():
            a = got[c].to_numpy()
            if a.dtype.kind == "f" or b.dtype.kind == "f":
                assert np.array_equal(a.astype(np.float64), b.astype(np.float64), equal_nan=True), (case, c, a[:5], b[:5])
            else:
                assert (a == b).all(), (case, c, a[:5], b[:5])
        assert sum(violations.values()) == n_printed, (case, violations, n_printed)
        rows += len(wl.df)
    return rows


def save(outs):
    arrays = {}
    for case, (cols, n_printed) in enumerate(outs):
        arrays[f"{case}/columns"] = np.array(list(cols))
        arrays[f"{case}/printed"] = np.array(n_printed)
        for i, v in enumerate(cols.values()):
            arrays[f"{case}/{i}"] = v
    np.savez_compressed(GOLDEN, **arrays)


def load():
    with np.load(GOLDEN) as z:
        n = len({k.split("/")[0] for k in z.files})
        return [({c: z[f"{case}/{i}"] for i, c in enumerate(z[f"{case}/columns"].tolist())}, int(z[f"{case}/printed"])) for case in range(n)]


def main():
    if "--golden" in sys.argv:  # the reference's outputs as recorded by --record: no reference tree needed
        rows = check(load())
        print("ingest_columns equals the real reference's row walk (recorded outputs) on", rows, "rows of 12 random workloads")
        return 0
    want = reference_outputs()
    if "--record" in sys.argv:
        save(want)
    rows = check(want)
    print("ingest_columns equals the real reference's row walk on", rows, "rows of 12 random workloads")
    return 0


if __name__ == "__main__":
    sys.exit(main())
