"""The reference's answers, recorded: what the `ref` fixture returns where the compiled reference (oracle/_ref) is absent.

The unmodified reference library can only be built where its sources are; the suite runs elsewhere too.  So the answers it gave to the
calls the suite makes are kept under tests/golden/ref_calls.npz and replayed: a call is identified by the method name and a digest of its
arguments (arrays by dtype, shape and bytes), and returns the stored result.  A call whose answer was not recorded (its result was too large
to keep in the repository) skips the test that makes it, naming the call.

Recording: run the tests with the compiled reference present and B200CV_RECORD_REF=1; every call's result (up to RECORD_LIMIT bytes) is
written to tests/golden/ref_calls.npz at the end of the session.
"""
import hashlib
import json
import os

import numpy as np

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
RECORD_LIMIT = 1024              # bytes of result per call kept in the repository (the larger answers are not kept)


def _digest(h, v):
    if isinstance(v, np.ndarray):
        a = np.ascontiguousarray(v)
        h.update(b"A%s%r" % (a.dtype.str.encode(), a.shape))
        h.update(a.tobytes())
    elif isinstance(v, (list, tuple)):
        h.update(b"L%d" % len(v))
        for x in v:
            _digest(h, x)
    elif isinstance(v, dict):
        h.update(b"D%d" % len(v))
        for k in sorted(v):
            _digest(h, k)
            _digest(h, v[k])
    elif isinstance(v, np.generic):
        _digest(h, v.item())
    else:
        h.update(b"S" + repr(v).encode())


def call_key(name, args, kwargs):
    h = hashlib.sha1(name.encode())
    _digest(h, list(args))
    _digest(h, dict(kwargs))
    return h.hexdigest()


def _flatten(v, arrays):
    if isinstance(v, np.ndarray):
        arrays.append(v)
        return {"a": len(arrays) - 1}
    if isinstance(v, (list, tuple)):
        return {"t" if isinstance(v, tuple) else "l": [_flatten(x, arrays) for x in v]}
    if isinstance(v, np.generic):
        return {"v": v.item()}
    return {"v": v}


def _unflatten(s, arrays):
    if "a" in s:
        return arrays[s["a"]].copy()
    if "t" in s:
        return tuple(_unflatten(x, arrays) for x in s["t"])
    if "l" in s:
        return [_unflatten(x, arrays) for x in s["l"]]
    return s["v"]


class RecordingOracle:
    """forwards every call to the compiled reference and keeps the (small enough) results"""

    def __init__(self, real):
        self._real = real
        self.kind = real.kind
        self._rec = {}

    def __getattr__(self, name):
        fn = getattr(self._real, name)
        if not callable(fn):
            return fn

        def call(*args, **kwargs):
            out = fn(*args, **kwargs)
            arrays = []
            struct = _flatten(out, arrays)
            if sum(a.nbytes for a in arrays) <= RECORD_LIMIT and all(a.dtype != object for a in arrays):
                self._rec[call_key(name, args, kwargs)] = (struct, arrays)
            return out
        return call

    def save(self):
        entries, blob = _load(os.path.join(GOLDEN, "ref_calls.npz"))
        parts = [blob]
        off = len(blob)
        for key, (struct, arrays) in self._rec.items():
            meta = []
            for a in arrays:
                b = np.ascontiguousarray(a).tobytes()
                meta.append([a.dtype.str, list(a.shape), off, len(b)])
                parts.append(b)
                off += len(b)
            entries[key] = {"s": struct, "a": meta}
        np.savez_compressed(os.path.join(GOLDEN, "ref_calls.npz"), index=np.array(json.dumps(entries, sort_keys=True)),
                            blob=np.frombuffer(b"".join(parts), np.uint8))


def _load(path):
    """{call key: {"s": result structure, "a": [[dtype, shape, offset, nbytes], ...]}} and the byte blob the arrays live in"""
    if not os.path.exists(path):
        return {}, b""
    with np.load(path) as z:
        return json.loads(str(z["index"])), z["blob"].tobytes()


class ReplayOracle:
    """the recorded answers of the compiled reference"""

    kind = "ref"

    def __init__(self):
        self._entries, self._blob = _load(os.path.join(GOLDEN, "ref_calls.npz"))

    def __getattr__(self, name):
        if name.startswith("_"):
            raise AttributeError(name)

        def call(*args, **kwargs):
            e = self._entries.get(call_key(name, args, kwargs))
            if e is None:
                import pytest
                pytest.skip("reference answer to %s(...) not recorded in tests/golden (oracle/_ref not built)" % name)
            arrays = [np.frombuffer(self._blob, np.dtype(dt), int(np.prod(shape, dtype=np.int64)), off).reshape(shape)
                      for dt, shape, off, nb in e["a"]]
            return _unflatten(e["s"], arrays)
        return call
