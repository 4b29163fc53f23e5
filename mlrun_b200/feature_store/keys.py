"""Entity keys and timestamps as the device takes them: int64 nanoseconds, and 64-bit keys from one int column, two int32
columns or one string column (FNV-1a, b2s_hash_strings).  Shared by the point-in-time join (offline.py) and the windowed
aggregations of feature-set ingest (ingest.py), so that both encode a feature set's keys the same way."""

import numpy as np

from ..lowering import LoweringError
from .online import _hash_strings

_NAT = -(1 << 63)
_UNIT_NS = {"s": 10**9, "ms": 10**6, "us": 10**3, "ns": 1}


def _ns(series, what):
    """datetime64 column -> (int64 nanoseconds, unit), NaT as INT64_MIN; LoweringError for other dtypes"""
    dt = series.dtype
    if getattr(dt, "tz", None) is not None or dt.kind != "M":
        raise LoweringError(f"{what} has dtype {dt}: the as-of join takes tz-naive datetime64 timestamps")
    unit = np.datetime_data(dt)[0]
    if unit not in _UNIT_NS:
        raise LoweringError(f"{what} has unit {unit!r}: the as-of join takes s / ms / us / ns timestamps")
    raw = series.to_numpy().view(np.int64)
    f = _UNIT_NS[unit]
    nat_mask = raw == _NAT
    if f > 1 and (np.abs(raw[~nat_mask]) > np.iinfo(np.int64).max // f).any():
        raise LoweringError(f"{what} holds timestamps outside the nanosecond range")
    return np.where(nat_mask, _NAT, raw * f), unit


def _key_kind(frame, names, what):
    """-> "int" | "pair" | "str" for the key columns `names` of `frame`"""
    dts = [frame[k].dtype for k in names]
    if len(names) == 1 and dts[0].kind in "iu" and dts[0] != np.uint64:
        return "int"
    if len(names) == 2 and all(str(d) == "int32" for d in dts):
        return "pair"
    if len(names) == 1 and (dts[0] == object or str(dts[0]) in ("str", "string")):
        return "str"
    raise LoweringError(f"{what}: keys {names} of dtypes {[str(d) for d in dts]} are not lowered (one int32 / int64 column, two "
                        "int32 columns or one string column)")


def _encode_keys(frame, names, kind, what):
    if kind == "int":
        return frame[names[0]].to_numpy().astype(np.int64)
    if kind == "pair":
        hi, lo = (frame[k].to_numpy().astype(np.int64) for k in names)
        return (hi << 32) | (lo & 0xFFFFFFFF)
    col = frame[names[0]]
    if col.isna().any():
        raise LoweringError(f"{what}: missing values in the string key {names[0]!r}")
    return _hash_strings(col.to_numpy())
