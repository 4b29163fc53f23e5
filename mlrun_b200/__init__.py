"""mlrun_b200 -- an H100-native serving-graph engine behind the mlrun.serving plugin API.

    import mlrun_b200 as mlrun
    fn = mlrun.new_function("f", kind="serving")
    graph = fn.set_topology("flow", engine="sync")
    graph.to(Imputer(...)).to(OneHotEncoder(...)).to("*FeatureRowVotingEnsemble", ...)
    server = fn.to_mock_server()
    server.test(body={...})            # the reference's per-event contract
    server.run_batch(X, names=cols)    # the engine: one fused CUDA launch for the whole batch

Importing the package never touches CUDA; device work goes through `mlrun_b200._native`, which raises
loudly when `libb200serve.so` or a GPU is missing (there is no CPU fallback on the hot path).
"""

__version__ = "0.1.0"

from . import feature_store, serving  # noqa: E402,F401
from .serving import ServingRuntime, new_function  # noqa: E402,F401
