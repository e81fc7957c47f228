"""Recorded results of the reference implementation, for the tests that compare against it.

The reference libraries under oracle/_ref are built only where the reference sources are present.
Every result they return inside a test is recorded under tests/golden/reference/<test module>.npz,
keyed by the test and the order of the call within it.  Where the libraries are absent, the same
calls return the recorded results, so the comparisons run on every checkout; where they are present,
each live result is checked against its recording.

Arrays larger than a call's `max_bytes` are recorded as a SHA-256 of their bytes.  The comparisons
that meet them are bit for bit, so `same_array` decides them from the digest as it would from the
array.  To (re)record, with oracle/_ref built:

    MPL_RECORD_REFERENCE=1 python -m pytest tests
"""
from __future__ import annotations

import base64
import hashlib
import json
import os
from pathlib import Path

import numpy as np

DIR = Path(__file__).resolve().parent / "golden" / "reference"
RECORD = os.environ.get("MPL_RECORD_REFERENCE") == "1"
UNRECORDED = {"seconds"}  # wall-clock fields differ from run to run
INLINE_BYTES = 1024  # larger recorded arrays are stored as members of the .npz, where they compress better
_calls: dict[str, int] = {}
_files: dict[str, dict] = {}
_members: dict[str, np.ndarray] = {}  # content-addressed arrays of all loaded or recorded modules


class Digest:
    """Shape, dtype and SHA-256 of an array's bytes."""

    def __init__(self, shape, dtype, sha256):
        self.shape, self.dtype, self.sha256 = tuple(shape), str(dtype), str(sha256)

    @classmethod
    def of(cls, a):
        a = np.ascontiguousarray(a)
        return cls(a.shape, a.dtype.str, hashlib.sha256(a.tobytes()).hexdigest())

    def __eq__(self, other):
        return isinstance(other, Digest) and (self.shape, self.dtype, self.sha256) == (other.shape, other.dtype, other.sha256)

    def __repr__(self):
        return f"Digest(shape={self.shape}, dtype={self.dtype}, sha256={self.sha256[:16]}...)"


def same_array(a, b, what="", bits=False):
    """a == b element for element (bits: byte for byte, so -0.0 != 0.0); either side may be a Digest."""
    if isinstance(a, Digest) or isinstance(b, Digest):
        da = a if isinstance(a, Digest) else Digest.of(a)
        db = b if isinstance(b, Digest) else Digest.of(b)
        assert da == db, (what, da, db)
    elif bits:
        assert a.shape == b.shape and a.tobytes() == b.tobytes(), what
    else:
        np.testing.assert_array_equal(a, b, err_msg=str(what))


def _encode(obj, max_bytes):
    if isinstance(obj, np.ndarray):
        if max_bytes is not None and obj.nbytes > max_bytes:
            obj = Digest.of(obj)
        else:
            a = np.ascontiguousarray(obj)
            if a.nbytes > INLINE_BYTES:
                name = hashlib.sha256(a.dtype.str.encode() + repr(a.shape).encode() + a.tobytes()).hexdigest()
                _members[name] = a
                return {"member": name}
            return {"array": [list(a.shape), a.dtype.str, base64.b64encode(a.tobytes()).decode()]}
    if isinstance(obj, Digest):
        return {"digest": [list(obj.shape), obj.dtype, obj.sha256]}
    if isinstance(obj, dict):
        return {"dict": {str(k): _encode(v, max_bytes) for k, v in obj.items() if k not in UNRECORDED}}
    if isinstance(obj, (list, tuple)):
        return {"list": [_encode(v, max_bytes) for v in obj]}
    if isinstance(obj, np.generic):
        obj = obj.item()
    if isinstance(obj, float):
        return {"float": obj.hex()}
    if isinstance(obj, bytes):
        return {"bytes": obj.hex()}
    assert obj is None or isinstance(obj, (bool, int, str)), type(obj)
    return {"value": obj}


def _decode(node):
    (kind, v), = node.items()
    if kind == "array":
        shape, dtype, data = v
        return np.frombuffer(base64.b64decode(data), dtype=np.dtype(dtype)).reshape(shape).copy()
    if kind == "member":
        return _members[v]
    if kind == "digest":
        return Digest(*v)
    if kind == "dict":
        return {k: _decode(x) for k, x in v.items()}
    if kind == "list":
        return [_decode(x) for x in v]
    if kind == "float":
        return float.fromhex(v)
    if kind == "bytes":
        return bytes.fromhex(v)
    return v


def _load(module):
    """{call key: encoded result} of one test module (one compressed JSON document)."""
    if module not in _files:
        f = DIR / f"{module}.npz"
        _files[module] = {}
        if f.exists():
            z = np.load(f, allow_pickle=False)
            _files[module] = json.loads(str(z["records"]))
            _members.update({k: z[k] for k in z.files if k != "records"})
    return _files[module]


def _member_names(node):
    (kind, v), = node.items()
    if kind == "member":
        yield v
    elif kind == "dict":
        for x in v.values():
            yield from _member_names(x)
    elif kind == "list":
        for x in v:
            yield from _member_names(x)


def _current_call():
    """(test module, key of this call): the test's id plus the number of reference calls it made before."""
    cur = os.environ.get("PYTEST_CURRENT_TEST")
    if not cur:
        return None, None
    nodeid = cur.rsplit(" (", 1)[0]
    path, _, test = nodeid.partition("::")
    n = _calls.get(nodeid, 0)
    _calls[nodeid] = n + 1
    return Path(path).stem, f"{test}#{n}".replace("/", "_")


def reference(library: Path, live, max_bytes=256):
    """The reference's result of one call: live() where `library` (under oracle/_ref) exists, else the
    recording of this call.  Recorded calls return arrays above max_bytes as Digests (None: keep all)."""
    module, key = _current_call()
    if Path(library).exists():
        r = live()
        if module is None:
            return r
        enc = _encode(r, max_bytes)
        files = _load(module)
        if RECORD:
            files[key] = enc
            DIR.mkdir(parents=True, exist_ok=True)
            used = {m: _members[m] for e in files.values() for m in _member_names(e)}
            np.savez_compressed(DIR / f"{module}.npz", records=np.array(json.dumps(files, sort_keys=True)), **used)
        elif key in files:
            _assert_same_tree(_decode(enc), _decode(files[key]),
                              f"{module}::{key}: the reference's result differs from its recording")
        return r
    if module is None:
        raise FileNotFoundError(f"{library} is not built")
    files = _load(module)
    if key not in files:
        raise LookupError(f"no recorded reference result for {module}::{key} (tests/golden/reference/{module}.npz); "
                          "record it with MPL_RECORD_REFERENCE=1 where oracle/_ref is built")
    return _decode(files[key])


def _assert_same_tree(a, b, what):
    if isinstance(a, dict):
        assert isinstance(b, dict) and a.keys() == b.keys(), what
        for k in a:
            _assert_same_tree(a[k], b[k], f"{what} [{k}]")
    elif isinstance(a, list):
        assert isinstance(b, list) and len(a) == len(b), what
        for i, (x, y) in enumerate(zip(a, b)):
            _assert_same_tree(x, y, f"{what} [{i}]")
    elif isinstance(a, (np.ndarray, Digest)):
        same_array(a, b, what, bits=True)
    else:
        assert a == b or (a != a and b != b), (what, a, b)
