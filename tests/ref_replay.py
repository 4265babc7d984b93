"""Record / replay of a session with the reference package, so that a check written against the live reference can run
from stored outputs where the reference is not installed.

`Recorder(module)` wraps a reference module: every top-level operation on it or on an object it hands out (attribute
access, call, indexing) runs for real, and its outcome is appended to a log — data (arrays, numbers, strings, enum
members by name, tuples of these) by value, anything else as an opaque object, an exception by its type name.  Each
call and index is logged with a digest of its arguments.  Calls made by the reference itself while it runs (e.g. into
a user constraint holding a wrapped object) are not logged.
`Replayer(log)` plays the log back for the same sequence of operations without the reference: it returns the stored
data, raises the stored exceptions, and fails loudly (`ReplayOutOfStep`) if the caller's sequence of operations or the
arguments of a call differ from the recorded ones (e.g. a problem generator changed after the recording).  `save_logs` / `load_logs` store per-key logs as one npz (arrays + a JSON skeleton, no pickle)."""
import builtins
import enum
import hashlib
import json

import numpy as np


class ReplayOutOfStep(BaseException):
    """The replayed caller did something else than the recorded one (BaseException: no `except Exception` swallows it)."""


class Named(object):
    """Replayed enum member: its type name and name are stored; one object per member, so identity checks still hold."""
    _members = {}

    def __new__(cls, etype, name):
        key = (etype, name)
        if key not in cls._members:
            obj = object.__new__(cls)
            obj.etype, obj.name = etype, name
            cls._members[key] = obj
        return cls._members[key]


_OBJ = {"k": "obj"}


def _is_data(v):
    if v is None or isinstance(v, (bool, int, float, str, np.ndarray, np.generic, enum.Enum)):
        return True
    return isinstance(v, (tuple, list)) and all(_is_data(x) for x in v)


def _digest(v, h):
    """Feeds a canonical form of call arguments into hash `h`; wrapped reference objects and other opaque objects (user
    classes, callbacks) count by kind only."""
    if isinstance(v, (Recorder, Replayer)):
        h.update(b"<ref>")
    elif isinstance(v, (enum.Enum, Named)):
        h.update(("E:%s;" % v.name).encode())
    elif isinstance(v, np.ndarray):
        h.update(("A%s%r:" % (v.dtype.str, v.shape)).encode())
        h.update(np.ascontiguousarray(v).tobytes())
    elif v is None or isinstance(v, (bool, int, float, str, np.generic)):
        h.update(("%s:%r;" % (type(v).__name__, v)).encode())
    elif isinstance(v, (list, tuple)):
        h.update(b"[")
        for x in v:
            _digest(x, h)
        h.update(b"]")
    elif isinstance(v, dict):
        for k in sorted(v):
            h.update(("%s=" % k).encode())
            _digest(v[k], h)
    else:
        h.update(("<%s>" % type(v).__name__).encode())


def _args_op(op, *args):
    h = hashlib.sha256()
    _digest(args, h)
    return "%s %s" % (op, h.hexdigest()[:16])


class _Log(object):
    def __init__(self):
        self.entries, self.depth = [], 0


def _unwrap(v):
    if isinstance(v, Recorder):
        return object.__getattribute__(v, "_real")
    if isinstance(v, list):
        return [_unwrap(x) for x in v]
    if isinstance(v, tuple):
        return tuple(_unwrap(x) for x in v)
    if isinstance(v, dict):
        return {k: _unwrap(x) for k, x in v.items()}
    return v


class Recorder(object):
    def __init__(self, real, log=None):
        object.__setattr__(self, "_real", real)
        object.__setattr__(self, "_log", log if log is not None else _Log())

    @property
    def log(self):
        return object.__getattribute__(self, "_log").entries

    def _do(self, op, fn):
        log = object.__getattribute__(self, "_log")
        if log.depth:                                   # the reference calling back into a wrapped object: transparent
            return fn()
        log.depth += 1
        try:
            out = fn()
        except Exception as e:
            log.entries.append((op, {"k": "raise", "type": type(e).__name__, "msg": str(e)[:200]}))
            raise
        finally:
            log.depth -= 1
        if _is_data(out):
            log.entries.append((op, {"k": "data", "v": out}))
            return out
        log.entries.append((op, _OBJ))
        return Recorder(out, log)

    def __getattr__(self, name):
        real = object.__getattribute__(self, "_real")
        return self._do("getattr " + name, lambda: getattr(real, name))

    def __call__(self, *args, **kwargs):
        real = object.__getattribute__(self, "_real")
        return self._do(_args_op("call", args, kwargs), lambda: real(*_unwrap(args), **_unwrap(kwargs)))

    def __getitem__(self, key):
        real = object.__getattribute__(self, "_real")
        return self._do(_args_op("getitem", key), lambda: real[_unwrap(key)])

    def __mro_entries__(self, bases):                    # `class C(wrapped_reference_class)` subclasses the real class
        return (object.__getattribute__(self, "_real"),)


class _ReplayBase(object):
    def __init__(self, *args, **kwargs):
        pass


class Replayer(object):
    def __init__(self, entries, pos=None):
        object.__setattr__(self, "_entries", entries)
        object.__setattr__(self, "_pos", pos if pos is not None else [0])

    def _next(self, op):
        entries, pos = object.__getattribute__(self, "_entries"), object.__getattribute__(self, "_pos")
        if pos[0] >= len(entries) or entries[pos[0]][0] != op:
            raise ReplayOutOfStep("replay step %d: caller did %r, the recorded session %r"
                                  % (pos[0], op, entries[pos[0]][0] if pos[0] < len(entries) else "(end)"))
        out = entries[pos[0]][1]
        pos[0] += 1
        if out["k"] == "data":
            return out["v"]
        if out["k"] == "raise":
            exc = getattr(builtins, out["type"], None)
            if not (isinstance(exc, type) and issubclass(exc, Exception)):
                exc = RuntimeError
            raise exc("replayed: %s" % out["msg"])
        return Replayer(entries, pos)

    def done(self):
        entries, pos = object.__getattribute__(self, "_entries"), object.__getattribute__(self, "_pos")
        return pos[0] == len(entries)

    def __getattr__(self, name):
        return self._next("getattr " + name)

    def __call__(self, *args, **kwargs):
        return self._next(_args_op("call", args, kwargs))

    def __getitem__(self, key):
        return self._next(_args_op("getitem", key))

    def __mro_entries__(self, bases):
        return (_ReplayBase,)


# ---- storage: {key: [(op, outcome), ...]} <-> npz (arrays concatenated per dtype, UTF-8 JSON skeleton, no pickle) --------
def _enc(v, flat):
    if isinstance(v, enum.Enum):
        return {"enum": v.name, "etype": type(v).__name__}
    if isinstance(v, Named):
        return {"enum": v.name, "etype": v.etype}
    if isinstance(v, np.generic):
        return {"np": v.dtype.str, "v": v.item()}
    if isinstance(v, np.ndarray):
        chunks = flat.setdefault(v.dtype.str, [])
        off = sum(c.size for c in chunks)
        chunks.append(np.ascontiguousarray(v).ravel())
        return {"a": v.dtype.str, "off": off, "shape": list(v.shape)}
    if isinstance(v, (tuple, list)):
        return {"seq": [_enc(x, flat) for x in v], "tuple": isinstance(v, tuple)}
    return {"py": v}


def _dec(d, flat):
    if "enum" in d:
        return Named(d["etype"], d["enum"])
    if "np" in d:
        return np.dtype(d["np"]).type(d["v"])
    if "a" in d:
        n = int(np.prod(d["shape"], dtype=np.int64))
        return flat[d["a"]][d["off"]:d["off"] + n].reshape(d["shape"]).copy()
    if "seq" in d:
        seq = [_dec(x, flat) for x in d["seq"]]
        return tuple(seq) if d["tuple"] else seq
    return d["py"]


def save_logs(path, logs):
    flat, skel = {}, {}
    for key, entries in logs.items():
        skel[key] = [[op, dict(out, v=_enc(out["v"], flat)) if out["k"] == "data" else out] for op, out in entries]
    arrays = {"flat%d" % i: np.concatenate(chunks) for i, chunks in enumerate(flat.values())}
    skel = {"logs": skel, "dtypes": {dt: "flat%d" % i for i, dt in enumerate(flat)}}
    np.savez_compressed(path, skeleton=np.frombuffer(json.dumps(skel).encode(), dtype=np.uint8), **arrays)


def load_logs(path):
    npz = np.load(path, allow_pickle=False)
    skel = json.loads(npz["skeleton"].tobytes().decode())
    flat = {dt: npz[name] for dt, name in skel["dtypes"].items()}
    return {key: [(op, dict(out, v=_dec(out["v"], flat)) if out["k"] == "data" else out) for op, out in entries]
            for key, entries in skel["logs"].items()}
