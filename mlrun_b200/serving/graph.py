"""Serving-graph topology and the per-event executors of the H100 engine.

Plugin-API mirror of mlrun/serving/states.py: the same step kinds, builder calls (`to`, `add_step`,
`add_route`, `error_handler`, `respond`, `set_flow`), wire format (`to_dict` / `from_dict`) and per-event
semantics (TaskStep.run :564-599, FlowStep.run :1279-1323, check_and_process_graph :1073-1184,
_init_async_objects :1622-1710), re-implemented around two ideas:

  * binding: `init_object` turns every step into ONE callable `step._invoke(event) -> event` that
    already knows its calling convention (full event / body, input_path / result_path, context
    injection, error handler), so the executors are plain loops over callables;
  * lowering: a run of recognised steps (feature transforms, device model servers, routers over them)
    is compiled by `mlrun_b200.serving.compiler` into a DevicePlan; batches take that plan, single
    events keep the per-step contract below.

The async engine is an in-process DAG walk (fan-out to every outlet, responder resolves the reply,
recovery steps) -- the observable contract of the storey flow the reference builds -- executed on
the caller's thread: there is no emit/await thread hand-off to pay for.
"""

import copy
import inspect
import os
import traceback

from .paths import merge_result, select_input
from .resolve import GraphError, MLRunInvalidArgumentError, err_to_str, get_class, get_function
from .serde import Serde, StepDict

MAX_ALLOWED_STEPS = 4500
QUEUE_NAMES = (">>", "$queue")
_TASK_FIELDS = ["kind", "class_name", "class_args", "handler", "skip_context", "after", "function", "comment",
                "shape", "full_event", "on_error", "responder", "input_path", "result_path"]


class StepKinds:
    router = "router"
    task = "task"
    flow = "flow"
    queue = "queue"
    choice = "choice"
    root = "root"
    error_step = "error_step"


def _step_name(name, class_name):
    if name:
        return name
    if not class_name:
        raise MLRunInvalidArgumentError("name or class_name must be provided")
    return class_name.__name__ if isinstance(class_name, type) else class_name


def _current_function(context):
    return (getattr(context, "current_function", None) or "") if context else ""


class BaseStep(Serde):
    kind = "BaseStep"
    default_shape = "ellipse"
    _dict_fields = ["kind", "comment", "after", "on_error"]

    def __init__(self, name=None, after=None, shape=None):
        self.name = name
        self.after = after or []
        self.shape = shape
        self.comment = None
        self.context = None
        self.on_error = None
        self._parent = None
        self._next = None
        self._error_call = None

    # ---- wiring ---------------------------------------------------------------------------------
    @property
    def next(self):
        return self._next

    @property
    def parent(self):
        return self._parent

    def set_parent(self, parent):
        self._parent = parent

    def set_next(self, key):
        if not self._next:
            self._next = [key]
        elif key not in self._next:
            self._next.append(key)
        return self

    def after_step(self, *after, append=True):
        if not append:
            self.after = []
        for item in after:
            item = item if isinstance(item, str) else item.name
            if item not in self.after:
                self.after.append(item)
        return self

    @property
    def fullname(self):
        name = self.name or ""
        if self._parent is not None and self._parent.fullname:
            name = f"{self._parent.fullname}/{name}"
        return name.replace(":", "_")

    def path_to_step(self, path):
        node = self
        for part in (path or "").split("/"):
            if part not in node:
                raise GraphError(f"step {part} doesnt exist in the graph under {node.fullname}")
            node = node[part]
        return node

    def get_children(self):
        return []

    def __iter__(self):
        return iter(())

    def _is_local_function(self, context):
        return True

    def supports_termination(self):
        return False

    # ---- builder --------------------------------------------------------------------------------
    def to(self, class_name=None, name=None, handler=None, graph_shape=None, function=None, full_event=None,
           input_path=None, result_path=None, **class_args):
        parent = self if hasattr(self, "steps") else self._parent
        if parent is None:
            raise GraphError(f"step {self.name} parent is not set or it's not part of a graph")
        name, step = params_to_step(class_name, name, handler, graph_shape=graph_shape, function=function,
                                    full_event=full_event, input_path=input_path, result_path=result_path,
                                    class_args=class_args)
        step = parent._steps.update(name, step)
        step.set_parent(parent)
        if parent is not self:
            step.after_step(self.name)
        parent._last_added = step
        return step

    def error_handler(self, name=None, class_name=None, handler=None, before=None, function=None, full_event=None,
                      input_path=None, result_path=None, **class_args):
        if not (class_name or handler):
            raise MLRunInvalidArgumentError("class_name or handler must be provided")
        if isinstance(self, RootFlowStep) and before:
            raise MLRunInvalidArgumentError("`before` arg can't be specified for graph error handler")
        name = _step_name(name, class_name)
        step = ErrorStep(class_name, class_args, handler, name=name, function=function, full_event=full_event,
                         input_path=input_path, result_path=result_path)
        self.on_error = name
        step.before = ([before] if isinstance(before, str) else before) or []
        step.base_step = self.name
        owner = self._parent if getattr(self, "_parent", None) is not None else self
        step = owner._steps.update(name, step)
        step.set_parent(owner)
        return self

    def set_flow(self, steps, force=False):
        raise NotImplementedError("set_flow() can only be called on a FlowStep")

    # ---- init / errors --------------------------------------------------------------------------
    def init_object(self, context, namespace, mode="sync", reset=False, **extra):
        self.context = context

    def _bind_error_handler(self):
        if self.on_error:
            self._error_call = self.context.root.path_to_step(self.on_error).run

    def _report(self, event, err, **kw):
        text = err_to_str(err)
        self.context.logger.error(f"step {self.name} got error {text} when processing an event:\n {event.body}")
        trace = traceback.format_exc()
        self.context.logger.error(trace)
        self.context.push_error(event, f"{text}\n{trace}", source=self.fullname, **kw)

    def _divert(self, event, err):
        if not event.error:
            event.error = {}
        event.error[self.name] = err_to_str(err)
        event.origin_state = self.fullname
        return self._error_call(event)


class TaskStep(BaseStep):
    kind = "task"
    _dict_fields = _TASK_FIELDS
    _default_class = ""

    def __init__(self, class_name=None, class_args=None, handler=None, name=None, after=None, full_event=None,
                 function=None, responder=None, input_path=None, result_path=None):
        super().__init__(name, after)
        self.class_name = class_name
        self.class_args = class_args or {}
        self.handler = handler
        self.function = function
        self.responder = responder
        self.full_event = full_event
        self.input_path = input_path
        self.result_path = result_path
        self.skip_context = None
        self._handler = None
        self._object = None
        self._class_object = None
        self._inject_context = False
        self._call_with_event = False
        self._node = None

    # ---- binding --------------------------------------------------------------------------------
    def init_object(self, context, namespace, mode="sync", reset=False, **extra):
        self.context = context
        self._node = None
        if not self._is_local_function(context):
            return
        if self.handler and not self.class_name:
            if callable(self.handler):
                self._handler, self.handler = self.handler, self.handler.__name__
            else:
                self._handler = get_function(self.handler, namespace)
            try:
                params = inspect.signature(self._handler).parameters
            except (TypeError, ValueError):
                params = {}
            self._inject_context = "context" in params
            self._bind_error_handler()
            return

        cls = self.class_name
        if isinstance(cls, type):
            self._class_object, self.class_name = cls, cls.__name__
        elif self._class_object is None:
            self._class_object = get_class(cls or self._default_class, namespace)
        if self._object is None or reset:
            try:
                self._object = self._class_object(**self._ctor_args(namespace, extra))
            except TypeError as exc:
                raise TypeError(f"failed to init step {self.name}\n args={self.class_args}") from exc
            chosen = self.handler
            if chosen:
                if not hasattr(self._object, chosen):
                    raise GraphError(f"handler ({chosen}) specified but doesnt exist in class {self.class_name}")
            elif hasattr(self._object, "do_event"):
                chosen, self._call_with_event = "do_event", True
            elif hasattr(self._object, "do"):
                chosen = "do"
            self._handler = getattr(self._object, chosen, None) if chosen else None
        self._bind_error_handler()
        if mode != "skip":
            self._post_init(mode)

    def _ctor_args(self, namespace, extra):
        """class_args (+ `_x` callables resolved) + the common args the class signature accepts"""
        args = {}
        for key, val in self.class_args.items():
            if key.startswith("_"):
                args[key[1:]] = get_function(val, namespace)
            else:
                args[key] = val
        args.update(extra)
        spec = inspect.getfullargspec(self._class_object)
        for key in ("name", "context", "input_path", "result_path", "full_event"):
            if spec.varkw or key in spec.args:
                args[key] = getattr(self, key)
        if spec.varkw or "graph_step" in spec.args:
            args["graph_step"] = self
        return args

    def _post_init(self, mode="sync"):
        if self._object is not None and hasattr(self._object, "post_init"):
            self._object.post_init(mode)

    def _is_local_function(self, context):
        current = _current_function(context)
        if current == "*" or (not self.function and not current):
            return True
        return self.function == "*" or (bool(self.function) and self.function == current) or self.function == current

    @property
    def async_object(self):
        return self._object

    def clear_object(self):
        self._object = None

    def respond(self):
        self.responder = True
        return self

    # ---- per-event call -------------------------------------------------------------------------
    def run(self, event, *args, **kwargs):
        if not self._is_local_function(self.context):
            return event
        if self._inject_context:
            kwargs["context"] = self.context
        else:
            kwargs.pop("context", None)
        try:
            if self.full_event or self._call_with_event:
                return self._handler(event, *args, **kwargs)
            if self._handler is None:
                raise MLRunInvalidArgumentError(f"step {self.name} does not have a handler")
            result = self._handler(select_input(self.input_path, event.body), *args, **kwargs)
            event.body = merge_result(self.result_path, event.body, result)
        except Exception as exc:
            if self._error_call is None:
                raise
            self._report(event, exc)
            recovered = self._divert(event, exc)  # first: the handler may replace event.body, and the merge below reads it after
            event.body = merge_result(self.result_path, event.body, recovered)
        return event


class ErrorStep(TaskStep):
    kind = "error_step"
    _dict_fields = _TASK_FIELDS + ["before", "base_step"]

    def __init__(self, *args, **kwargs):
        super().__init__(*args, **kwargs)
        self.before = None
        self.base_step = None


class RouterStep(TaskStep):
    kind = "router"
    default_shape = "doubleoctagon"
    _dict_fields = _TASK_FIELDS + ["routes"]
    _default_class = "mlrun.serving.ModelRouter"

    def __init__(self, class_name=None, class_args=None, handler=None, routes=None, name=None, function=None,
                 input_path=None, result_path=None):
        super().__init__(class_name, class_args, handler, name=name, function=function, input_path=input_path,
                         result_path=result_path)
        self._routes = None
        self.routes = routes

    @property
    def routes(self):
        return self._routes

    @routes.setter
    def routes(self, routes):
        self._routes = StepDict.from_dict(CLASSES, routes, "task")

    def get_children(self):
        return self._routes.values()

    def add_route(self, key, route=None, class_name=None, handler=None, function=None, **class_args):
        if not route and not class_name and not handler:
            raise MLRunInvalidArgumentError("route or class_name must be specified")
        if not route:
            route = TaskStep(class_name, class_args, handler=handler)
        route.function = function or route.function
        if len(self._routes) >= MAX_ALLOWED_STEPS:
            raise MLRunInvalidArgumentError(
                f"Cannot create the serving graph: the maximum number of steps is {MAX_ALLOWED_STEPS}")
        route = self._routes.update(key, route)
        route.set_parent(self)
        return route

    def clear_children(self, routes=None):
        for key in list(routes or self._routes.keys()):
            del self._routes[key]

    def init_object(self, context, namespace, mode="sync", reset=False, **extra):
        if not self._is_local_function(context):
            return
        self.class_args = self.class_args or {}
        super().init_object(context, namespace, "skip", reset=reset, routes=self._routes, **extra)
        for route in self._routes.values():
            if self.function and not route.function:
                route.function = self.function
            route.set_parent(self)
            route.init_object(context, namespace, mode, reset=reset)
        self._bind_error_handler()
        self._post_init(mode)

    def __getitem__(self, name):
        return self._routes[name]

    def __setitem__(self, name, route):
        self.add_route(name, route)

    def __delitem__(self, key):
        del self._routes[key]

    def __iter__(self):
        return iter(self._routes.keys())

    def __contains__(self, name):
        return name in self._routes


class QueueStep(BaseStep):
    """queue / stream hop.  Mock servers run multi-function graphs in-process: a queue with downstream
    steps is an identity (states.py:1638, 1675-1676); with a path it pushes to the stream and terminates"""

    kind = "queue"
    default_shape = "cds"
    _dict_fields = BaseStep._dict_fields + ["path", "shards", "retention_in_hours", "trigger_args", "options"]

    def __init__(self, name=None, path=None, after=None, shards=None, retention_in_hours=None, trigger_args=None, **options):
        super().__init__(name, after)
        self.path = path
        self.shards = shards
        self.retention_in_hours = retention_in_hours
        self.trigger_args = trigger_args
        self.options = options
        self._stream = None
        self._node = None

    def init_object(self, context, namespace, mode="sync", reset=False, **extra):
        self.context = context
        if self.path:
            from .host import get_stream_pusher

            self._stream = get_stream_pusher(self.path, **self.options)
        self._bind_error_handler()

    @property
    def async_object(self):
        return self._node

    def to(self, class_name=None, name=None, handler=None, graph_shape=None, function=None, full_event=None,
           input_path=None, result_path=None, **class_args):
        if not function:
            raise MLRunInvalidArgumentError(
                f"step '{_step_name(name, class_name)}' must specify a function, because it follows a queue step")
        return super().to(class_name, name, handler, graph_shape, function, full_event, input_path, result_path, **class_args)

    def run(self, event, *args, **kwargs):
        if event.body and self._stream is not None:
            self._stream.push(event.body)
            event.terminated = True
            event.body = None
        return event


class FlowStep(BaseStep):
    kind = "flow"
    _dict_fields = BaseStep._dict_fields + ["steps", "engine", "default_final_step"]

    def __init__(self, name=None, steps=None, after=None, engine=None, final_step=None):
        super().__init__(name, after)
        self._steps = None
        self.steps = steps
        self.engine = engine
        self.final_step = final_step
        self.from_step = os.environ.get("START_FROM_STEP", None)
        self._last_added = None
        self._start_steps = []
        self._dag = None
        self._wait_for_result = False
        self._controller = None

    @property
    def steps(self):
        return self._steps

    @steps.setter
    def steps(self, steps):
        self._steps = StepDict.from_dict(CLASSES, steps, "task")

    @property
    def controller(self):
        return self._controller

    def get_children(self):
        return self._steps.values()

    def is_empty(self):
        return len(self._steps) == 0

    def __getitem__(self, name):
        return self._steps[name]

    def __setitem__(self, name, step):
        self.add_step(name, step)

    def __delitem__(self, key):
        del self._steps[key]

    def __iter__(self):
        return iter(self._steps.keys())

    def __contains__(self, name):
        return name in self._steps

    # ---- builder --------------------------------------------------------------------------------
    def add_step(self, class_name=None, name=None, handler=None, after=None, before=None, graph_shape=None,
                 function=None, full_event=None, input_path=None, result_path=None, **class_args):
        name, step = params_to_step(class_name, name, handler, graph_shape=graph_shape, function=function,
                                    full_event=full_event, input_path=input_path, result_path=result_path,
                                    class_args=class_args)
        for item in after if isinstance(after, list) else [after]:
            self.insert_step(name, step, item, before)
        return step

    def insert_step(self, key, step, after, before=None):
        step = self._steps.update(key, step)
        step.set_parent(self)
        if after == "$prev" and len(self._steps) == 1:
            after = None
        previous = ""
        if after:
            if after == "$prev" and self._last_added is not None:
                previous = self._last_added.name
            elif after not in self._steps:
                raise MLRunInvalidArgumentError(f"cant set after, there is no step named {after}")
            else:
                previous = after
            step.after_step(previous)
        if before:
            if before not in self._steps:
                raise MLRunInvalidArgumentError(f"cant set before, there is no step named {before}")
            if before in (step.name, previous):
                raise GraphError(f"graph loop, step {before} is specified in before and/or after {key}")
            self[step.name].after_step(*self[before].after, append=False)
            self[before].after_step(step.name, append=False)
        self._last_added = step
        return step

    def clear_children(self, steps=None):
        for key in list(steps or self._steps.keys()):
            del self._steps[key]

    def set_flow(self, steps, force=False):
        if not force and self.steps:
            raise MLRunInvalidArgumentError(
                "set_flow() called on a step that already has downstream steps. "
                "If you want to overwrite existing steps, set force=True.")
        self.steps = None
        step = self
        for item in steps:
            step = step.to(**item) if isinstance(item, dict) else step.to(item)
        return step

    def list_child_functions(self):
        found = []
        for step in self.get_children():
            fn = getattr(step, "function", None)
            if fn and fn not in found:
                found.append(fn)
        return found

    def supports_termination(self):
        return self.engine != "sync"

    # ---- init -----------------------------------------------------------------------------------
    def init_object(self, context, namespace, mode="sync", reset=False, **extra):
        self.context = context
        for name, step in self._steps.items():  # error steps claim their place in the DAG first
            if step.kind == StepKinds.error_step:
                self._place_error_step(name, step)
        self.check_and_process_graph()
        for step in self._steps.values():
            step.set_parent(self)
            step.init_object(context, namespace, mode, reset=reset)
        self._bind_error_handler()
        if self.engine != "sync":
            self._dag, self._wait_for_result = _build_dag(self, context)
            self._controller = _InlineController(self._dag, context)

    def _place_error_step(self, name, step):
        if not step.before and not any(step.name in other.after for other in self._steps.values()):
            step.responder = True
            return
        for target in step.before:
            if target not in self._steps:
                raise MLRunInvalidArgumentError(f"cant set before, there is no step named {target}")
            self[target].after_step(name)

    def check_and_process_graph(self, allow_empty=False):
        """validate the DAG, set `.next` links, pick start steps / default final step / responders"""
        if self.is_empty() and allow_empty:
            self._start_steps = []
            return [], None, []

        def loop_from(step, seen):
            for prev in step.after or []:
                if prev in seen:
                    return step.name
                hit = loop_from(self[prev], seen + [prev])
                if hit:
                    return hit
            return None

        starts = []
        for step in self._steps.values():
            step._next = None
            if step.after:
                bad = loop_from(step, [])
                if bad:
                    raise GraphError(f"Error, loop detected in step {bad}, graph must be acyclic (DAG)")
            else:
                starts.append(step.name)
        responders = []
        for step in self._steps.values():
            if getattr(step, "responder", None) and step.kind != StepKinds.error_step:
                responders.append(step.name)
            if step.on_error and step.on_error in starts:
                starts.remove(step.on_error)
            for prev in step.after or []:
                self[prev].set_next(step.name)
        if self.on_error and self.on_error in starts:
            starts.remove(self.on_error)
        if len(responders) > 1:
            raise GraphError(f'there are more than one responder steps in the graph ({",".join(responders)})')
        if self.from_step:
            if self.from_step not in self.steps:
                raise GraphError(f"from_step ({self.from_step}) specified and not found in graph steps")
            starts = [self.from_step]
        self._start_steps = [self[n] for n in starts]

        current = _current_function(self.context)
        if current and current != "*":
            def first_of(step):
                if getattr(step, "function", None) == current:
                    return step
                for item in step.next or []:
                    hit = first_of(self[item])
                    if hit:
                        return hit
                return None

            narrowed = [s for s in (first_of(st) for st in self._start_steps) if s]
            if not narrowed:
                raise GraphError(f"did not find steps pointing to current function ({current})")
            self._start_steps = narrowed
        if self.engine == "sync" and len(self._start_steps) > 1:
            raise GraphError("sync engine can only have one starting step (without .after)")

        final = None
        if self.final_step:
            if self.final_step not in self.steps:
                raise GraphError(f"final_step ({self.final_step}) specified and not found in graph steps")
            final = self.final_step
        elif len(self._start_steps) == 1:
            cur = self._start_steps[0]
            while cur is not None:
                if not cur.next:
                    final = cur.name
                    break
                cur = self[cur.next[0]] if len(cur.next) == 1 else None
        return self._start_steps, final, responders

    # ---- per-event executors --------------------------------------------------------------------
    def run(self, event, *args, **kwargs):
        if self._controller is not None:
            reply = self._controller.emit(event, self._wait_for_result)
            if self._wait_for_result and reply is not None:
                return reply
            event = copy.copy(event)
            event.body = {"id": event.id}
            return event
        if not self._start_steps:
            return event
        cur = self._start_steps[0]
        while cur is not None:
            try:
                event = cur.run(event, *args, **kwargs)
            except Exception as exc:
                if self._error_call is None:
                    raise
                self._report(event, exc, failed_step=cur.name)
                event.body = self._divert(event, exc)
                event.terminated = True
                return event
            if getattr(event, "terminated", None):
                return event
            if isinstance(getattr(event, "error", None), dict) and cur.name in event.error:
                cur = self._steps[cur.on_error]
            nxt = cur.next
            if nxt and len(nxt) > 1:
                raise GraphError(f"synchronous flow engine doesnt support branches use async, step={cur.name}")
            cur = self[nxt[0]] if nxt else None
        return event

    def wait_for_completion(self):
        if self._controller is not None:
            self._controller.terminate()
            return self._controller.await_termination()


class RootFlowStep(FlowStep):
    kind = "root"
    _dict_fields = ["steps", "engine", "final_step", "on_error"]


CLASSES = {"task": TaskStep, "router": RouterStep, "flow": FlowStep, "queue": QueueStep, "error_step": ErrorStep}


def graph_root_setter(server, graph):
    if not graph:
        return
    if isinstance(graph, dict):
        kind = graph.get("kind")
    elif hasattr(graph, "kind"):
        kind = graph.kind
    else:
        raise MLRunInvalidArgumentError("graph must be a dict or a valid object")
    if kind == StepKinds.router:
        server._graph = server._verify_dict(graph, "graph", RouterStep)
    elif not kind or kind == StepKinds.root:
        server._graph = server._verify_dict(graph, "graph", RootFlowStep)
    else:
        raise GraphError(f"illegal root step {kind}")


def params_to_step(class_name, name, handler=None, graph_shape=None, function=None, full_event=None,
                   input_path=None, result_path=None, class_args=None):
    """step object from the builder arguments: objects with `to_dict`, "*Router", ">>"/"$queue", class / handler"""
    class_args = class_args or {}
    if class_name and hasattr(class_name, "to_dict"):
        struct = class_name.to_dict()
        kind = struct.get("kind", StepKinds.task)
        name = name or struct.get("name", struct.get("class_name"))
        step = CLASSES.get(kind, RootFlowStep).from_dict(struct)
        step.function = function
        step.full_event = full_event or step.full_event
        step.input_path = input_path or step.input_path
        step.result_path = result_path or step.result_path
        if hasattr(class_name, "_b200_keep_instance"):
            step._live_object = class_name  # declarative transforms can be lowered from the live object
    elif class_name and class_name in QUEUE_NAMES:
        if "path" not in class_args:
            raise MLRunInvalidArgumentError("path=<stream path or None> must be specified for queues")
        if not name:
            raise MLRunInvalidArgumentError("queue name must be specified")
        if full_event is not None:
            class_args = dict(class_args, full_event=full_event)
        step = QueueStep(name, **class_args)
    elif class_name and isinstance(class_name, str) and class_name.startswith("*"):
        routes = class_args.get("routes", None)
        class_name = class_name[1:]
        name = _step_name(name, class_name or "router")
        step = RouterStep(class_name, class_args, handler, name=name, function=function, routes=routes,
                          input_path=input_path, result_path=result_path)
    elif class_name or handler:
        name = _step_name(name, class_name)
        step = TaskStep(class_name, class_args, handler, name=name, function=function, full_event=full_event,
                        input_path=input_path, result_path=result_path)
    else:
        raise MLRunInvalidArgumentError("class_name or handler must be provided")
    if graph_shape:
        step.shape = graph_shape
    return name, step


# ================================================================================= async engine
from .merger import DROP  # noqa: E402


def _branch_copy(event):
    """an extra outlet gets its own deep copy of the payload (storey's fan-out contract: branches never see each other's
    in-place edits; tests/serving/test_merger.py:107-128)"""
    ev = copy.copy(event)
    ev.body = copy.deepcopy(event.body)
    return ev


class _Node:
    __slots__ = ("name", "fullname", "call", "full_event", "input_path", "result_path", "kwargs", "outlets",
                 "recovery", "completes")

    def __init__(self, name, call=None, full_event=False, input_path=None, result_path=None, kwargs=None, completes=False):
        self.name = name
        self.fullname = name
        self.call = call
        self.full_event = full_event
        self.input_path = input_path
        self.result_path = result_path
        self.kwargs = kwargs or {}
        self.outlets = []
        self.recovery = None
        self.completes = completes


class _Reply:
    __slots__ = ("event", "set")

    def __init__(self):
        self.event = None
        self.set = False


class _InlineController:
    """emit() walks the DAG on the caller's thread and returns the responder's event"""

    def __init__(self, starts, context):
        self.starts = starts
        self.context = context

    def emit(self, event, want_reply):
        reply = _Reply()
        for i, node in enumerate(self.starts):
            self._visit(node, event if i == 0 else copy.copy(event), reply)
        return reply.event if (want_reply and reply.set) else None

    def _visit(self, node, event, reply):
        if node.completes:
            if not reply.set:
                reply.event, reply.set = event, True
            return
        try:
            if node.full_event:
                out = node.call(event, **node.kwargs)
                if out is DROP:
                    return
                out = event if out is None else out
            else:
                result = node.call(select_input(node.input_path, event.body), **node.kwargs)
                if result is DROP:
                    return
                out = copy.copy(event)
                out.body = merge_result(node.result_path, event.body, result)
        except Exception as exc:
            if node.recovery is None:
                raise
            if not getattr(event, "error", None):
                event.error = {}
            event.error[node.name] = err_to_str(exc)
            event.origin_state = node.fullname
            self._visit(node.recovery, event, reply)
            return
        payloads = [out] + [_branch_copy(out) for _ in node.outlets[1:]]  # copied before any branch runs
        for outlet, ev in zip(node.outlets, payloads):
            self._visit(outlet, ev, reply)

    def terminate(self):
        pass

    def await_termination(self):
        return None


def _build_dag(flow, context):
    """one node per local step; native (MapClass-style) step objects keep their own call convention"""
    trigger = getattr(context, "trigger", None)
    can_respond = trigger is None or trigger == "http"
    wait_for_result = False
    for step in flow._steps.values():
        step._node = None
        if not (hasattr(step, "async_object") and step._is_local_function(context)):
            continue
        if step.kind == StepKinds.queue:
            stream = step._stream
            if step.path and not (context.is_mock and step.next) and stream is not None:
                node = _Node(step.name, call=lambda body, _s=stream: (_s.push(body), body)[1])
            else:
                node = _Node(step.name, call=lambda body: body)
        else:
            obj = step._object
            if obj is not None and getattr(obj, "_native_step", False) and hasattr(obj, "do"):
                node = _Node(step.name, call=obj.do, full_event=bool(getattr(obj, "_full_event", None)),
                             input_path=getattr(obj, "_input_path", None), result_path=getattr(obj, "_result_path", None))
            else:
                node = _Node(step.name, call=step._handler, full_event=bool(step.full_event or step._call_with_event),
                             input_path=step.input_path, result_path=step.result_path,
                             kwargs={"context": context} if step._inject_context else None)
        node.fullname = step.fullname
        step._node = node
        if can_respond and not step.next and getattr(step, "responder", None):
            node.outlets.append(_Node("complete", completes=True))
            wait_for_result = True

    seen = set()

    def link(step):
        if step.name in seen or not step._is_local_function(context):
            return
        seen.add(step.name)
        for item in step.next or []:
            nxt = flow[item]
            if getattr(nxt, "_node", None) is not None:
                step._node.outlets.append(nxt._node)
                link(nxt)

    starts = []
    for step in flow._start_steps:
        if getattr(step, "_node", None) is not None:
            starts.append(step._node)
            link(step)
    for step in flow._steps.values():
        node = getattr(step, "_node", None)
        target = step.on_error or flow.on_error
        if node is None or not target:
            continue
        err_step = flow._steps[target]
        if err_step is step or getattr(err_step, "_node", None) is None:
            continue
        node.recovery = err_step._node
        for item in err_step.next or []:
            nxt = getattr(flow[item], "_node", None)
            if nxt is not None and nxt not in err_step._node.outlets:
                err_step._node.outlets.append(nxt)
    return starts, wait_for_result
