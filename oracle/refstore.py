"""Stored outputs of the reference's own code, for machines where oracle/_ref/ cannot be built.

The entry points of oracle/binding.py that run the reference's compiled sources (the ref_* functions, RefOrb, and the matchers
with impl="ref") are wrapped by `recorded`.  Where the library exists in oracle/_ref/ they call it.  Elsewhere they answer from
tests/golden/refcalls/*.npz: what the reference returned for exactly these arguments, found by a hash of the arguments.  A call
whose arguments were never recorded raises MissingRecord, so a comparison with the reference is never skipped quietly.

Recording: run the tests with PLSLAM_REF_RECORD=<dir> where oracle/_ref/ is built; at exit every wrapped call made is written to
<dir>/<library>_<function>.npz (added to what that file already holds).  Copy the files into tests/golden/refcalls/.
"""
import atexit
import functools
import glob
import hashlib
import inspect
import json
import os

import numpy as np

GOLDEN = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden", "refcalls")
_index = None       # key -> path of the .npz that holds it
_open = {}          # path -> np.lib.npyio.NpzFile
_recorded = {}      # file stem -> {key: (spec, arrays)}
_context = {}       # state the reference keeps between calls (the last Frame constructed, the image a RefOrb last saw)


class MissingRecord(KeyError):
    pass


def _digest(h, v):
    if hasattr(v, "_ref_args"):                       # a RefOrb: its constructor arguments
        v = v._ref_args
    if isinstance(v, (np.ndarray, np.generic)):
        a = np.ascontiguousarray(v)
        h.update(f"a{a.dtype.descr}{a.shape}".encode())
        h.update(a.tobytes())
    elif isinstance(v, (list, tuple)):
        h.update(f"l{len(v)}".encode())
        for x in v:
            _digest(h, x)
    elif isinstance(v, dict):
        h.update(f"d{len(v)}".encode())
        for k in sorted(v, key=repr):
            h.update(repr(k).encode())
            _digest(h, v[k])
    else:                                             # None, bool, int, float, str
        h.update(f"{type(v).__name__}:{v!r}".encode())


def _flatten(v, key, arrays):
    if isinstance(v, tuple):
        return {"tuple": [_flatten(x, key, arrays) for x in v]}
    if isinstance(v, dict):
        return {"dict": {k: _flatten(x, key, arrays) for k, x in v.items()}}
    if isinstance(v, (np.ndarray, np.generic)):
        name = f"{key}.{len(arrays)}"
        arrays[name] = np.asarray(v)
        return {"array": name, "scalar": isinstance(v, np.generic)}
    assert v is None or isinstance(v, (bool, int, float, str)), type(v)
    return {"value": v}


def _unflatten(spec, npz):
    if "tuple" in spec:
        return tuple(_unflatten(x, npz) for x in spec["tuple"])
    if "dict" in spec:
        return {k: _unflatten(x, npz) for k, x in spec["dict"].items()}
    if "array" in spec:
        a = npz[spec["array"]]
        return a[()] if spec["scalar"] else a
    return spec["value"]


def has(library):
    return bool(glob.glob(os.path.join(GOLDEN, f"{library}_*.npz")))


def _lookup(key):
    global _index
    if _index is None:
        _index = {}
        for path in sorted(glob.glob(os.path.join(GOLDEN, "*.npz"))):
            with np.load(path) as z:
                for k in z.files:
                    if "." not in k:
                        _index[k] = path
    path = _index.get(key)
    if path is None:
        raise MissingRecord(f"no stored reference output for {key}: record it with PLSLAM_REF_RECORD where oracle/_ref/ is built")
    if path not in _open:
        _open[path] = np.load(path)
    z = _open[path]
    return _unflatten(json.loads(str(z[key])), z)


def _write(out_dir):
    os.makedirs(out_dir, exist_ok=True)
    for stem, calls in _recorded.items():
        path = os.path.join(out_dir, stem + ".npz")
        data = {}
        if os.path.exists(path):
            with np.load(path) as z:
                data = {k: z[k] for k in z.files}
        for key, (spec, arrays) in calls.items():
            data[key] = np.array(json.dumps(spec))
            data.update(arrays)
        np.savez_compressed(path, **data)


def recorded(library, lib_path, uses=None, sets=None):
    """Wrap an entry point that runs the reference's code in the library lib_path.  `uses` / `sets` name reference state a call
    reads / leaves behind (its key then includes / becomes that state)."""
    def deco(f):
        sig = inspect.signature(f)
        name = f.__qualname__.replace(".", "_")

        @functools.wraps(f)
        def call(*args, **kw):
            bound = sig.bind(*args, **kw)
            bound.apply_defaults()
            if bound.arguments.get("impl", "ref") != "ref":
                return f(*args, **kw)
            h = hashlib.sha1()
            _digest(h, dict(bound.arguments))
            if uses:
                h.update(_context.get(uses, "").encode())
            key = f"{name}-{h.hexdigest()}"
            if sets:
                _context[sets] = key
            if not os.path.exists(lib_path):
                return _lookup(key)
            out = f(*args, **kw)
            rec = os.environ.get("PLSLAM_REF_RECORD")
            if rec:
                if not _recorded:
                    atexit.register(_write, rec)
                arrays = {}
                spec = _flatten(out, key, arrays)
                _recorded.setdefault(f"{library}_{name}", {})[key] = (spec, arrays)
            return out
        return call
    return deco
