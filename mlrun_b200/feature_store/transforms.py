"""Feature-store transform steps of the H100 engine (plugin-API mirror of mlrun.feature_store.steps).

Each step is *declarative*: it holds the same constructor arguments as the reference class
(mlrun/feature_store/steps.py) and is lowered by `mlrun_b200.lowering.ColumnProgram` into a device
plan when it sits in a run of recognised steps over numeric columns -- that is the hot path.

`do(event)` keeps the reference's per-event call contract for everything the device cannot hold
(string / object values, a lone step between user Python steps): it is host-side *plugin
compatibility*, evaluated with plain Python on one dict, and is never used for batches (a batched
body that cannot be lowered raises instead of falling back -- see GraphServer.run_batch).
"""

import math
import re
import uuid

import numpy as np

from ..serving.resolve import MLRunInvalidArgumentError
from ..serving.step_meta import StepMeta


def _is_missing(v):
    # what pd.isna() answers for the scalar kinds an event can carry (None, NaN, NaT, pd.NA)
    if v is None:
        return True
    if isinstance(v, float):
        return math.isnan(v)
    name = type(v).__name__
    if name in ("NaTType", "NAType"):
        return True
    try:
        return bool(v != v)  # numpy floats / datetimes that are NaN/NaT
    except Exception:
        return False


class _Step(StepMeta):
    """common kwargs every reference step accepts through storey.MapClass"""

    def __init__(self, context=None, name=None, full_event=None, input_path=None, result_path=None, **kwargs):
        self.context = context
        self.name = name
        self._full_event = full_event
        self._input_path = input_path
        self._result_path = result_path
        self._kwargs = kwargs
        self.logger = getattr(context, "logger", None) if context else None
        self._native_step = True  # tells the async engine to honour the step's own call convention

    def do(self, event):
        body = event.body if hasattr(event, "body") and self._full_event else event
        if hasattr(body, "columns") and hasattr(body, "index"):
            raise TypeError(
                f"{type(self).__name__}: DataFrame bodies are not processed on the host; "
                "send a float32 matrix through GraphServer.run_batch / the device plan"
            )
        return self._do_event(event)


class Imputer(_Step):
    """steps.py:377-413 -- NaN/None -> mapping.get(feature, default_value) for every feature"""

    def __init__(self, method="avg", default_value=None, mapping=None, **kwargs):
        super().__init__(**kwargs)
        self.mapping = mapping or {}
        self.method = method
        self.default_value = default_value

    def _do_event(self, event):
        m, d = self.mapping, self.default_value
        return {k: (m.get(k, d) if _is_missing(v) else v) for k, v in event.items()}


class OneHotEncoder(_Step):
    """steps.py:427-513 -- mapped features are replaced in place by 0/1 fields, one per category"""

    def __init__(self, mapping, **kwargs):
        super().__init__(**kwargs)
        for key, values in mapping.items():
            for val in values:
                if not isinstance(val, (str, int, np.integer)):  # a bool is an int here too, as in the reference
                    raise MLRunInvalidArgumentError("For OneHotEncoder you must provide int or string mapping list")
            mapping[key] = list(dict.fromkeys(values))
        self.mapping = mapping

    @staticmethod
    def _sanitized_category(category):
        return re.sub("[ -]", "_", category) if isinstance(category, str) else category

    def _do_event(self, event):
        out = {}
        for feature, value in event.items():
            cats = self.mapping.get(feature)
            if not cats:
                out[feature] = value
                continue
            for c in cats:
                out[f"{feature}_{self._sanitized_category(c)}"] = 0
            if value in cats:
                out[f"{feature}_{self._sanitized_category(value)}"] = 1
            elif self.logger:
                self.logger.warn(f"OneHotEncoder does not have an encoding for value '{value}' of feature '{feature}'")
        return out


class MapValues(_Step):
    """steps.py:152-216 -- value / range replacement; only mapped features survive unless with_original_features"""

    def __init__(self, mapping, with_original_features=False, suffix="mapped", **kwargs):
        super().__init__(**kwargs)
        self.mapping = mapping
        self.with_original_features = with_original_features
        self.suffix = suffix

    @classmethod
    def validate_args(cls, feature_set, **kwargs):
        """ingest-time check of the constructor arguments (steps.py:331-370): one value type per column (NaN aside), and
        ranges never next to single replacements"""
        for column, rules in kwargs.get("mapping", []).items():  # QUIRK: no mapping at all is an AttributeError ([] has no items)
            if "ranges" in rules:
                if len(rules) > 1:
                    raise MLRunInvalidArgumentError("MapValues - mapping values of the same column can not combine ranges and "
                                                    f"single replacement, which is the case for column '{column}'")
                values = [v for pair in rules["ranges"].values() for v in pair if v != "-inf" and v != "inf"]
            else:
                values = list(rules.values())
            kinds = {type(v) for v in values if not (isinstance(v, (float, np.floating)) and math.isnan(v))}
            if len(kinds) > 1:
                raise MLRunInvalidArgumentError("MapValues - mapping values of the same column must be in the same type, which "
                                                f"was not the case for Column '{column}'")

    def _map_value(self, feature, value):
        fmap = self.mapping.get(feature, {})
        for label, bounds in fmap.get("ranges", {}).items() if "ranges" in fmap else ():
            lo = -math.inf if bounds[0] == "-inf" else bounds[0]
            hi = math.inf if bounds[1] == "inf" else bounds[1]
            if value >= lo and value < hi:  # operand order as upstream (same TypeError text for non-numbers)
                return label
        return fmap.get(value, value)

    def _do_event(self, event):
        key = (lambda f: f"{f}_{self.suffix}") if self.with_original_features else (lambda f: f)
        out = {key(f): self._map_value(f, v) for f, v in event.items() if f in self.mapping}
        if self.with_original_features:
            out.update(event)
        return out


class DropFeatures(_Step):
    """steps.py:699-735"""

    def __init__(self, features, **kwargs):
        super().__init__(**kwargs)
        self.features = features

    @classmethod
    def validate_args(cls, feature_set, **kwargs):
        """entities, the label column and the timestamp key are not features (steps.py:737-753)"""
        features = kwargs.get("features", [])
        spec = feature_set.spec
        entities = set(features) & set(spec.entities.keys())
        if entities:
            raise MLRunInvalidArgumentError(f"DropFeatures can only drop features, not entities: {entities}")
        for what, name in (("label_column", spec.label_column), ("timestamp_key", spec.timestamp_key)):
            if name in features:
                raise MLRunInvalidArgumentError(f"DropFeatures can not drop {what}: {name}")

    def _do_event(self, event):
        for f in self.features:
            if f not in event:
                raise MLRunInvalidArgumentError(f"The ingesting data doesn't contain a feature named '{f}'")
            del event[f]
        return event


class DateExtractor(_Step):
    """steps.py:516-602 -- pandas-style date parts of `timestamp_col` as new `<col>_<part>` fields"""

    def __init__(self, parts, timestamp_col=None, **kwargs):
        super().__init__(**kwargs)
        self.timestamp_col = timestamp_col or "timestamp"
        self.parts = parts

    def _do_event(self, event):
        import pandas as pd

        if self.timestamp_col not in event:
            raise MLRunInvalidArgumentError(f"{self.timestamp_col} does not exist in the event")
        ts = pd.Timestamp(event[self.timestamp_col])
        for part in self.parts:
            event[f"{self.timestamp_col}_{part}"] = getattr(ts, part)
        return event


class SetEventMetadata(_Step):
    """steps.py:635-696 -- copy id / key from the body onto the event"""

    def __init__(self, id_path=None, key_path=None, random_id=None, **kwargs):
        kwargs["full_event"] = True
        super().__init__(**kwargs)
        self.id_path = id_path
        self.key_path = key_path
        self.random_id = random_id

    def post_init(self, mode="sync"):
        """part of the step protocol (the reference builds its tagging closures here); the paths are read in `do`"""

    def do(self, event):
        from ..serving.paths import get_in

        if self.id_path:
            event.id = str(get_in(event.body, self.id_path))
        if self.key_path:
            event.key = str(get_in(event.body, self.key_path))
        if self.random_id:
            event.id = uuid.uuid4().hex
        return event


class FeaturesetValidator(_Step):
    """steps.py:94-128 -- range checks that only report; events pass through unchanged"""

    def __init__(self, featureset=None, columns=None, name=None, validators=None, **kwargs):
        kwargs["full_event"] = True
        super().__init__(name=name, **kwargs)
        self.featureset = featureset or "."
        self.columns = columns
        self._validators = dict(validators or {})
        self.violations = 0

    def do(self, event):
        body = event.body
        for name, v in self._validators.items():
            if name in body:
                ok, args = v.check(body[name])
                if not ok:
                    self.violations += 1
                    message = args.pop("message")
                    key_text = f" key={event.key}" if getattr(event, "key", None) else ""
                    print(f"{v.severity}! {name} {message},{key_text} args={args}")
        return event
