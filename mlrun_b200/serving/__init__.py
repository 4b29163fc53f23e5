"""mlrun_b200.serving -- drop-in names of mlrun.serving, backed by the H100 engine"""
from .device_models import (  # noqa: F401
    FeatureRowModelServer,
    FeatureRowVotingEnsemble,
    LGBMModelServer,
    PickleModelServer,
    SKLearnModelServer,
    XGBoostModelServer,
)
from .events import MockEvent, MockTrigger, Response  # noqa: F401
from .function import ServingFunction, ServingRuntime, new_function  # noqa: F401
from .graph import (  # noqa: F401
    ErrorStep,
    FlowStep,
    QueueStep,
    RootFlowStep,
    RouterStep,
    StepKinds,
    TaskStep,
)
from .host import GraphContext, GraphServer, create_graph_server, nuclio_init_hook, v2_serving_handler, v2_serving_init  # noqa: F401
from .model_server import V2ModelServer  # noqa: F401
from .resolve import GraphError, MLRunInvalidArgumentError  # noqa: F401
from .routing import ModelRouter, ParallelRun, ParallelRunnerModes, VotingEnsemble, VotingTypes  # noqa: F401

# the reference's module paths (`from mlrun.serving.routers import VotingEnsemble`, `mlrun.serving.server.MockEvent`,
# `mlrun.serving.states.RouterStep`, `mlrun.serving.v2_serving.V2ModelServer`) resolve to the modules that
# hold those names here -- aliases in sys.modules, not copies
import sys as _sys  # noqa: E402

from . import graph as _graph  # noqa: E402
from . import host as _host  # noqa: E402
from . import merger as _merger  # noqa: E402,F401
from . import model_server as _model_server  # noqa: E402
from . import routing as _routing  # noqa: E402

for _alias, _module in (("routers", _routing), ("states", _graph), ("server", _host), ("v2_serving", _model_server)):
    _sys.modules.setdefault(f"{__name__}.{_alias}", _module)
    globals().setdefault(_alias, _module)
