"""Serving host of the H100 engine: GraphContext, GraphServer, mock streams, nuclio-style hooks.

Plugin-API mirror of mlrun/serving/server.py (GraphServer :86-312, v2_serving_init/handler :315-409,
create_graph_server :412-434, GraphContext :493-602).  On top of the reference surface the server
exposes the batched entry points of the engine:

    server.device_plan          the DevicePlan the whole graph lowered to (None + .lowering_error otherwise)
    server.run_batch(X)         (B, F) float32 rows -> outputs, one fused CUDA launch, no per-event Python
    server.run_events(bodies)   list of feature-dict bodies -> list of per-event responses; rows whose
                                status word is non-zero come back as 400 Responses, like a failing event
"""

import asyncio
import json
import os
import socket
import traceback

import numpy as np

from .codec import BINARY_CONTENT_TYPE
from .events import MockEvent, MockTrigger, Response  # noqa: F401
from .graph import RootFlowStep, RouterStep, graph_root_setter  # noqa: F401
from .resolve import MLRunInvalidArgumentError, caller_globals, err_to_str, get_function, logger as _logger
from .serde import Serde

SERVING_SPEC_ENV = "SERVING_SPEC_ENV"
EVENT_ID_HEADER = "MLRUN-EVENT-ID"
EVENT_PATH_HEADER = "MLRUN-EVENT-PATH"
_STREAM_TRIGGERS = ("kafka", "kafka-cluster", "v3ioStream", "v3io-stream", "rabbit-mq", "rabbitMq")


def _json_default(obj):
    if isinstance(obj, np.ndarray):
        return obj.tolist()
    if isinstance(obj, np.generic):
        return obj.item()
    return str(obj)


class _DummyStream:
    """`dummy://` stream: keeps pushed records in .event_list (mlrun/datastore/__init__.py:115-127)"""

    def __init__(self, event_list=None, **kwargs):
        self.event_list = [] if event_list is None else event_list

    def push(self, data, **kwargs):
        self.event_list.extend(data if isinstance(data, list) else [data])


class _MockQueueStream:
    """`v3io://...` with stream_args={"mock": True}: records {"data": json} in ._mock_queue"""

    def __init__(self, **kwargs):
        self._mock_queue = []

    def push(self, data, **kwargs):
        for rec in data if isinstance(data, list) else [data]:
            self._mock_queue.append({"data": rec if isinstance(rec, (str, bytes)) else json.dumps(rec, default=_json_default)})


def get_stream_pusher(stream_path, **kwargs):
    if stream_path.startswith("dummy://"):
        return _DummyStream(event_list=kwargs.get("event_list"))
    if stream_path.startswith("v3io") and kwargs.get("mock"):
        return _MockQueueStream()
    raise ValueError(f"unsupported stream path {stream_path}: this engine ships dummy:// and mocked v3io streams only")


class _StreamContext:
    def __init__(self, enabled, parameters, function_uri):
        self.enabled = False
        self.hostname = socket.gethostname()
        self.function_uri = function_uri
        self.output_stream = None
        self.stream_uri = None
        log_stream = parameters.get("log_stream", "")
        if (enabled or log_stream) and function_uri:
            self.enabled = True
            project = function_uri.split("/")[0] if "/" in function_uri else "default"
            self.stream_uri = log_stream.format(project=project) if log_stream else f"dummy://{project}"
            self.output_stream = get_stream_pusher(self.stream_uri, **parameters.get("stream_args", {}))


class GraphContext:
    def __init__(self, level="info", logger=None, server=None, nuclio_context=None):
        self.state = None
        self.logger = logger
        self.worker_id = 0
        self.Response = Response
        self.verbose = False
        self.stream = None
        self.root = None
        if nuclio_context is not None:
            self.logger = nuclio_context.logger
            self.Response = nuclio_context.Response
            if hasattr(getattr(nuclio_context, "trigger", None), "kind"):
                self.trigger = nuclio_context.trigger.kind
            self.worker_id = nuclio_context.worker_id
            if hasattr(nuclio_context, "platform"):
                self.platform = nuclio_context.platform
        elif logger is None:
            self.logger = _logger
        self._server = server
        self.current_function = None
        self.get_store_resource = None
        self.get_table = None
        self.is_mock = False
        self.monitoring_mock = False

    @property
    def server(self):
        return self._server

    @property
    def project(self):
        uri = (self._server.function_uri if self._server else "") or ""
        return uri.split("/")[0] if "/" in uri else ""

    def push_error(self, event, message, source=None, **kwargs):
        if self.verbose:
            self.logger.error(f"got error from {source} state:\n{event.body}\n{message}")
        stream = getattr(self._server, "_error_stream_object", None) if self._server else None
        if stream is None:
            return
        try:
            stream.push({"function_uri": self._server.function_uri, "worker": self.worker_id, "host": socket.gethostname(),
                         "source": source, "event": {"id": event.id, "body": event.body}, "message": message, "args": kwargs})
        except Exception as exc:  # noqa: BLE001
            self.logger.error(f"failed to write to error stream: {exc}\n{traceback.format_exc()}")

    def get_param(self, key, default=None):
        if self._server is not None and self._server.parameters:
            return self._server.parameters.get(key, default)
        return default

    def get_secret(self, key):
        return None


class GraphServer(Serde):
    kind = "server"

    def __init__(self, graph=None, parameters=None, load_mode=None, function_uri=None, verbose=False, version=None,
                 functions=None, graph_initializer=None, error_stream=None, track_models=None, tracking_policy=None,
                 secret_sources=None, default_content_type=None):
        self._graph = None
        self.graph = graph
        self.function_uri = function_uri
        self.parameters = parameters or {}
        self.verbose = verbose
        self.load_mode = load_mode or "sync"
        self.version = version or "v2"
        self.context = None
        self._current_function = None
        self.functions = functions or {}
        self.graph_initializer = graph_initializer
        self.error_stream = error_stream
        self.track_models = track_models
        self.tracking_policy = tracking_policy
        self._error_stream_object = None
        self.secret_sources = secret_sources
        self.default_content_type = default_content_type
        self.http_trigger = True
        self._compiled = None

    @property
    def graph(self):
        return self._graph

    @graph.setter
    def graph(self, graph):
        graph_root_setter(self, graph)

    def set_current_function(self, function):
        self._current_function = function

    def set_error_stream(self, error_stream):
        self.error_stream = error_stream
        self._error_stream_object = get_stream_pusher(error_stream) if error_stream else None

    def init_states(self, context, namespace, resource_cache=None, logger=None, is_mock=False, monitoring_mock=False):
        if self.error_stream:
            self._error_stream_object = get_stream_pusher(self.error_stream)
        ctx = GraphContext(server=self, nuclio_context=context, logger=logger)
        ctx.is_mock = is_mock
        ctx.monitoring_mock = monitoring_mock
        ctx.root = self.graph
        ctx.stream = _StreamContext(self.track_models, self.parameters, self.function_uri)
        ctx.current_function = self._current_function
        ctx.verbose = self.verbose
        self.context = ctx
        if self.graph_initializer:
            init = self.graph_initializer if callable(self.graph_initializer) else get_function(self.graph_initializer, namespace or [])
            init(self)
        ctx.root = self.graph

    def init_object(self, namespace):
        self.graph.init_object(self.context, namespace, self.load_mode, reset=True)
        self._compiled = None

    # ---- reference per-event surface ------------------------------------------------------------
    def test(self, path="/", body=None, method="", headers=None, content_type=None, silent=False, get_body=True,
             event_id=None, trigger=None, offset=None, time=None):
        if not self.graph:
            raise MLRunInvalidArgumentError("no models or steps were set, use function.set_topology() and add steps")
        event = MockEvent(body=body, path=path, method=method or ("POST" if body else "GET"), headers=headers,
                          content_type=content_type, event_id=event_id, trigger=trigger, offset=offset, time=time)
        resp = self.run(event, get_body=get_body)
        if getattr(resp, "status_code", 0) >= 300 and not silent:
            raise RuntimeError(f"failed ({resp.status_code}): {resp.body}")
        return resp

    def run(self, event, context=None, get_body=False, extra_args=None):
        own = self.context
        context = context or own
        event.content_type = event.content_type or self.default_content_type or ""
        if event.headers:
            event.id = event.headers.get(EVENT_ID_HEADER, event.id)
            event.path = event.headers.get(EVENT_PATH_HEADER, event.path)
        if event.content_type == BINARY_CONTENT_TYPE and isinstance(event.body, (bytes, bytearray, memoryview)):
            # the engine's binary wire format: float32 rows in, 4-byte result words out, one fused launch (no JSON at all)
            try:
                return self.run_binary(event.body)
            except Exception as exc:  # noqa: BLE001 -- like any other failure of this event: its 400
                message = f"{type(exc).__name__}: {err_to_str(exc)}"
                own.push_error(event, message, source="_handler")
                return context.Response(body=message, content_type="text/plain", status_code=400)
        is_json = event.content_type in ("json", "application/json")
        if isinstance(event.body, (str, bytes)) and (not event.content_type or is_json):
            try:
                event.body = json.loads(event.body)
            except (json.decoder.JSONDecodeError, UnicodeDecodeError) as exc:
                if is_json:
                    message = f"failed to json decode event, {err_to_str(exc)}"
                    context.logger.error(message)
                    own.push_error(event, message, source="_handler")
                    return context.Response(body=message, content_type="text/plain", status_code=400)
        try:
            response = self.graph.run(event, **(extra_args or {}))
        except Exception as exc:  # noqa: BLE001 -- any step failure is this event's 400
            message = f"{type(exc).__name__}: {err_to_str(exc)}"
            if own.verbose:
                message += "\n" + traceback.format_exc()
            context.logger.error(f"run error, {traceback.format_exc()}")
            own.push_error(event, message, source="_handler")
            return context.Response(body=message, content_type="text/plain", status_code=400)
        if asyncio.iscoroutine(response):
            response = asyncio.get_event_loop().run_until_complete(response)
        body = response.body
        if get_body or isinstance(body, context.Response):
            return body
        if body and not isinstance(body, (str, bytes)):
            # strict, as upstream (server.py:303-304): a numpy value in a response is a TypeError for the caller
            return context.Response(body=json.dumps(body), content_type="application/json", status_code=200)
        return body

    def wait_for_completion(self):
        return self.graph.wait_for_completion() if hasattr(self.graph, "wait_for_completion") else None

    # ---- batched surface of the engine ----------------------------------------------------------
    def compile(self, in_names=None):
        """lower the whole graph into one DevicePlan (cached); raises LoweringError when it cannot"""
        from .compiler import compile_graph

        if self._compiled is None or (in_names is not None and list(in_names) != self._compiled.in_names):
            self._compiled = compile_graph(self.graph, in_names)
            # the function's engine parameters (fn.spec.parameters["b200"], handed over like every other parameter:
            # runtimes/nuclio/serving.py:668-724): the coalescing ring of this graph's plan
            ring = (self.parameters or {}).get("b200") or {}
            if ring and hasattr(self._compiled.plan, "set_ring"):
                unknown = set(ring) - {"max_batch", "max_wait_us", "ring_slots"}
                if unknown:
                    raise ValueError(f'parameters["b200"]: unknown keys {sorted(unknown)}')
                self._compiled.plan.set_ring(ring_slots=ring.get("ring_slots", 0), max_batch=ring.get("max_batch", 0),
                                             max_wait_us=ring.get("max_wait_us", -1))
        return self._compiled

    def emit(self, body):
        """one event body (a feature dict of the compiled schema) -> ticket.  The rows of concurrent callers are coalesced
        into one device batch by the plan's ring (`b2s_submit`): the replacement of storey's SyncEmitSource.emit
        (serving/states.py:1283-1287).  Collect the response with `await_result(ticket)`."""
        compiled = self.compile(list(body.keys()))
        return compiled.plan.submit(compiled.pack_events([body]))

    def await_result(self, ticket):
        """blocks until the ticket's batch ran; -> the response dict `run_events` gives that event (or its 400 Response)"""
        compiled = self.compile()
        out, status = compiled.plan.wait(ticket, with_status=True)
        return compiled.responses(out, status, self.context)[0]

    @property
    def device_plan(self):
        return self.compile().plan

    def run_batch(self, X, names=None, with_status=False):
        """(B, F) float32 rows, columns named `names` (default f0..fF-1 or the compiled schema) ->
        (B, out_cols) outputs from one fused launch.  Semantics: row i is the event {names[j]: X[i, j]}.

        Rows already in HBM are scored there; the outputs (and status words) then come back as `_native.DeviceArray`s,
        ready when returned, and the producer's queued writes are awaited first:
          - a CUDA matrix (a torch tensor, any DLPack or CUDA-array-interface producer, a DeviceArray such as
            `get_offline_tensors(...).features` with names=t.columns): float32, unit inner stride, a row stride that is a
            multiple of 4 bytes; read in place at its own row stride, without a copy.  Equals run_batch(X.cpu().numpy()).
          - a `columnar.DeviceColumnBatch` (its result and index columns) or a mapping of CUDA columns: `names` (default: the
            compiled schema) picks the plan's input columns in order; float32/64, (u)int8/16/32/64 and bool columns are
            packed into float32 rows on the device, each converted as `astype(np.float32)` converts it.  Equals, bit for bit,
            run_batch(np.stack([np.asarray(c).astype(np.float32) for c in picked], axis=1), names).  That can differ from
            `frame[names].to_numpy(np.float32)` of a mixed frame, which goes through float64 and so rounds an int64 above
            2**53 twice."""
        from ..feature_store import columnar

        if columnar.is_device_column(X):
            return self._run_device_matrix(X, names, with_status)
        if isinstance(X, (dict, columnar.DeviceColumnBatch)) and columnar.is_device_source(X):
            return self._run_device_columns(X, names, with_status)
        compiled = self.compile(names)
        return compiled.plan.run(np.ascontiguousarray(X, dtype=np.float32), with_status=with_status)

    def _run_device_matrix(self, X, names, with_status):
        """run_batch of a CUDA matrix: b2s_run_device over the rows where they are"""
        from ..feature_store.columnar import DeviceColumn
        from ..lowering import LoweringError
        from ..plan import check_rows

        m = DeviceColumn(X, "X", matrix=True)
        if m.dtype != np.float32:
            raise LoweringError(f"the CUDA matrix has dtype {m.dtype}: the plan reads float32 rows (build it with "
                                'get_offline_tensors(..., dtype="float32"))')
        if names is not None:
            check_rows(m, len(names))
        plan = self.compile(names).plan
        check_rows(m, plan.n_in)
        n = m.shape[0]
        stride = m.strides[0] if n > 1 else plan.n_in * 4  # one row: any stated stride reads the same words
        if stride % 4:
            raise ValueError(f"the CUDA matrix's row stride of {stride} bytes is not a multiple of 4")
        out, status = _device_results(plan, n, with_status)
        try:
            m.acquire()
            if m.ptr % 4:
                raise ValueError("the CUDA matrix does not start on a 4-byte boundary")
            if n:
                plan.run_device(m.ptr, n, stride, out.ptr, status.ptr if status is not None else None)
                _device_sync()
        finally:
            m.release()
        return (out, status) if with_status else out

    def _run_device_columns(self, X, names, with_status):
        """run_batch of CUDA columns: b2s_run_columns_device packs the picked columns into rows and scores them"""
        from .. import _native as nat
        from ..feature_store import columnar
        from ..feature_store.online import table_cols
        from ..lowering import LoweringError

        cols = columnar.device_columns(X)
        if len({c.n for c in cols.values()}) > 1:
            raise ValueError("All arrays must be of the same length")
        names = list(self.compile().in_names if names is None else names)
        for name in names:
            if name in cols and cols[name].dtype.kind == "M":
                raise LoweringError(f"feature {name!r} is a {cols[name].dtype} column: a matrix of numbers has no place for it "
                                    "(drop it from names)")
        picked = table_cols(cols, names, "feature")
        plan = self.compile(names).plan
        n = next(iter(cols.values())).n if cols else len(X)
        out, status = _device_results(plan, n, with_status)
        try:
            tcols = [nat.TableCol(c.acquire().ptr, dt.itemsize, kind) for c, dt, kind in picked]
            plan.run_columns_device(tcols, n, out.ptr, status.ptr if status is not None else None)
            _device_sync()
        finally:
            for c in cols.values():
                c.release()
        return (out, status) if with_status else out

    def run_events(self, bodies, path=None):
        """feature-dict event bodies -> per-event responses through the fused plan.  Rows flagged by the
        device (non-finite model input) come back as the 400 Response the reference would give that event."""
        from .model_server import now_date

        start = now_date()
        compiled = self.compile(list(bodies[0].keys()) if bodies else None)
        X = compiled.pack_events(bodies)
        out, status = compiled.plan.run(X, with_status=True)
        responses = compiled.responses(out, status, self.context)
        if compiled.tracker is not None:  # model tracking: the records per-event pushes would have produced
            ok = [i for i, r in enumerate(responses) if isinstance(r, dict)]
            compiled.tracker.push_batch(start, _Lazy(len(ok), lambda j: {"inputs": [X[ok[j]].tolist()]}),
                                        lambda j: responses[ok[j]], _tracked_op(compiled.tracker))
        return responses


    def run_enriched(self, keys, with_status=False):
        """batched enrichment + predict for a graph whose root is an Enrichment router: entity keys -> outputs with the
        online-table gather feeding the fused scoring plan on the device (`b2s_table_enrich_host`: keys in, votes and status
        words out, nothing else crosses PCIe); replaces EnrichmentVotingEnsemble.preprocess + the per-model predicts,
        serving/routers.py:1335-1342.  Unknown keys come back with status bit 4 (ROW_UNKNOWN_KEY).  CUDA keys (one int column,
        or a mapping of the vector's `index_keys` int columns) stay in HBM: the outputs and status words come back as
        `_native.DeviceArray`s, ready when returned."""
        from ..lowering import LoweringError

        compiled = self.compile()
        router = getattr(self.graph, "_object", None) if self.graph.kind == "router" else None
        svc = getattr(router, "_feature_service", None)
        if svc is None or not hasattr(svc, "table"):
            raise LoweringError("run_enriched needs an EnrichmentModelRouter / EnrichmentVotingEnsemble at the root")
        plan = compiled.plan
        if plan.n_in != svc.table.n_feat:
            raise LoweringError(f"the feature vector has {svc.table.n_feat} features, the models take {plan.n_in}")
        d_keys = svc._device_keys(keys)
        if d_keys is None:
            out, status = svc.table.enrich(plan, svc._encode_keys(keys))
        else:
            try:
                out, status = svc.table.enrich_arrays(plan, d_keys)
            finally:
                d_keys.release()
        return (out, status) if with_status else out

    def run_binary(self, body):
        """`application/x-b2s-f32` request (codec.encode_rows) -> Response carrying the outputs in the same format;
        a batch with a row the device flags answers 400 as a whole, like `run_json` (one event carries all rows)"""
        from . import codec

        X = codec.decode_rows(body)
        if X.dtype != np.float32:
            raise ValueError("the request words must be float32 feature values")
        out, status = self.compile().plan.run(np.ascontiguousarray(X), with_status=True)
        if status.any():
            return self.context.Response(body="ValueError: Input X contains NaN or infinity.", content_type="text/plain",
                                         status_code=400)
        return self.context.Response(body=codec.encode_rows(out), content_type=codec.BINARY_CONTENT_TYPE, status_code=200)

    def run_json(self, body, event_id=None):
        """wire-level batched entry for graphs whose root is a router / model server: a V2 body
        `{"inputs": [[...], ...]}` (bytes / str) -> the Response GraphServer.run would answer for it (serving/server.py:
        252-308), through the C body codec and ONE fused launch.  Bodies that are not a numeric matrix raise
        `codec.NotV2Matrix` (use `run` for them)."""
        import uuid

        from ..lowering import LoweringError
        from . import codec

        from .model_server import now_date

        start = now_date()
        compiled = self.compile()
        name, version = compiled.responder
        if not name:
            raise LoweringError("run_json needs a graph that ends in a model server or a voting ensemble")
        X, rest = codec.decode_body(body)
        out, status = compiled.plan.run(np.ascontiguousarray(X), with_status=True)
        if status.any():  # scikit-learn raises for the whole request (one event carries all rows)
            return self.context.Response(body="ValueError: Input X contains NaN or infinity.", content_type="text/plain",
                                         status_code=400)
        response = {"id": event_id or rest.get("id") or uuid.uuid4().hex, "model_name": name, "outputs": None}
        if version:
            response["model_version"] = version
        if compiled.tracker is not None:  # one request carrying all rows = one tracked event
            vals = out[:, 0] if out.shape[1] == 1 else out
            compiled.tracker.push_batch(start, _Lazy(1, lambda j: {"id": response["id"], "inputs": X.tolist(), **rest}),
                                        lambda j: {**response, "outputs": vals.tolist()}, _tracked_op(compiled.tracker))
        text = codec.format_outputs(out[:, 0] if out.shape[1] == 1 else out)
        return self.context.Response(body=codec.dumps_with_outputs(response, text), content_type="application/json", status_code=200)


def _device_results(plan, n, with_status):
    """the outputs (and, with_status, the status words) of n rows as DeviceArrays"""
    from .. import _native as nat

    out = nat.DeviceArray(nat.darray_alloc(max(n * plan.out_cols * 4, 4)), (n, plan.out_cols), plan.out_dtype)
    status = nat.DeviceArray(nat.darray_alloc(max(n * 4, 4)), (n,), np.int32) if with_status else None
    return out, status


def _device_sync():
    from .. import _native as nat

    nat.check(nat.load().b2s_device_sync())


def _tracked_op(tracker):
    """routers log their own events without an operation (routers.py:901-903), model servers with it (v2_serving.py:331-340)"""
    return None if hasattr(tracker.model, "routes") else "infer"


class _Lazy:
    """index -> record, built on demand (push_batch only materialises the sampled rows)"""

    def __init__(self, n, fn):
        self.n, self._fn = n, fn

    def __len__(self):
        return self.n

    def __call__(self, i):
        return self._fn(i)


def v2_serving_init(context, namespace=None):
    spec = json.loads(os.environ[SERVING_SPEC_ENV])
    server = GraphServer.from_dict(spec)
    if hasattr(context, "trigger"):
        server.http_trigger = getattr(context.trigger, "kind", "http") == "http"
    server.set_current_function(os.getenv("SERVING_CURRENT_FUNCTION", ""))
    ns = namespace or caller_globals()
    kw = {"is_mock": context.is_mock} if hasattr(context, "is_mock") else {}
    server.init_states(context, ns, **kw)
    server.init_object(ns)
    context.mlrun_handler = v2_serving_handler
    context._server = server


def nuclio_init_hook(context, data, kind):
    if kind != "serving_v2":
        raise ValueError("failed to init serving function, unsupported kind")
    v2_serving_init(context, data)


def v2_serving_handler(context, event, get_body=False):
    if context._server.http_trigger and event.body == b"":
        event.body = None
    event.stream_path = getattr(event, "topic", event.path)
    if hasattr(event, "trigger") and event.trigger.kind in _STREAM_TRIGGERS:
        event.path = "/"
    return context._server.run(event, context, get_body)


def create_graph_server(parameters=None, load_mode=None, graph=None, verbose=False, current_function=None, **kwargs):
    server = GraphServer(graph, parameters or {}, load_mode, verbose=verbose, **kwargs)
    server.set_current_function(current_function or os.getenv("SERVING_CURRENT_FUNCTION", ""))
    return server
