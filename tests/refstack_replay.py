"""Record / replay of every value that crosses the boundary between a test and the reference's Python stack.

tests/test_refpin_vector.py drives the reference's `gymnasium` / `metaworld` objects through `RefSession.module()`
proxies.  With the environment variable METAWORLD_REFERENCE pointing at a Meta-World checkout, the proxies wrap the
live reference (on oracle/refshim) and log, in order, every attribute read, call, item access, iteration and
raised exception, with the arguments the test passed; the log is written to tests/golden/refstack_<test>.pkl.gz.
Without it the proxies replay that log: each access must match the recorded one (same path, same arguments, compared
exactly) and returns the recorded value, so the test compares this package against the reference's outputs as they
were when the log was written, on any machine.

The fixtures `ref` (the test's session), `gym` and `metaworld` (the proxied modules) are shared by the test modules that
import them.
"""
import builtins
import gzip
import os
import pickle

import numpy as np
import pytest

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
_PLAIN = (type(None), bool, int, float, complex, str, bytes, np.generic, np.dtype)


class _Handle:
    """Stands in a log entry for a reference object the test keeps using (its later accesses have their own entries)."""

    def __init__(self, path):
        self.path = path

    def __eq__(self, other):
        return isinstance(other, _Handle) and other.path == self.path


class Box:
    """Recorded form of a gymnasium Box space."""

    def __init__(self, low, high, shape, dtype):
        self.low, self.high, self.shape, self.dtype = low, high, shape, dtype


def _is_task(v):
    return type(v).__name__ == "Task" and hasattr(v, "env_name") and hasattr(v, "data")


def _plain(v):
    if _is_task(v):             # a NamedTuple, but it unpickles only where the reference is importable
        return False
    if isinstance(v, _PLAIN):
        return True
    if isinstance(v, np.ndarray):
        return v.dtype != object or all(_plain(x) for x in v.flat)
    if isinstance(v, (list, tuple)):
        return all(_plain(x) for x in v)
    if isinstance(v, dict):
        return all(_plain(k) and _plain(x) for k, x in v.items())
    return False


def _same(a, b):
    if isinstance(a, np.ndarray) or isinstance(b, np.ndarray):
        a, b = np.asarray(a), np.asarray(b)
        if a.dtype == object or b.dtype == object:
            return a.shape == b.shape and all(_same(x, y) for x, y in zip(a.flat, b.flat))
        return a.dtype == b.dtype and a.shape == b.shape and np.array_equal(a, b, equal_nan=True)
    if isinstance(a, (list, tuple)) and isinstance(b, (list, tuple)):
        return len(a) == len(b) and all(_same(x, y) for x, y in zip(a, b))
    if isinstance(a, dict) and isinstance(b, dict):
        return a.keys() == b.keys() and all(_same(a[k], b[k]) for k in a)
    return type(a) is type(b) and a == b


class RefSession:
    def __init__(self, name):
        self.path = os.path.join(GOLD, f"refstack_{name}.pkl.gz")
        self.root = os.environ.get("METAWORLD_REFERENCE")
        self.recording = bool(self.root)
        if self.recording:
            self.log = []
        else:
            with gzip.open(self.path, "rb") as f:
                self.log = pickle.load(f)
            self.pos = 0

    def module(self, name):
        """The reference's `gymnasium` or `metaworld` module, behind a proxy."""
        if self.recording:
            from oracle import refshim
            refshim.activate(self.root)
            import importlib
            return _Proxy(self, name, importlib.import_module(name))
        return _Proxy(self, name, None)

    def close(self):
        if self.recording:
            with gzip.open(self.path, "wb", compresslevel=9) as f:
                pickle.dump(self.log, f, protocol=4)
        else:
            assert self.pos == len(self.log), f"the test stopped after {self.pos} of {len(self.log)} recorded reference accesses"

    # -- one access: `op` on `path` with `args`; `live` computes the reference's answer while recording
    def access(self, op, path, args, live):
        if self.recording:
            stored_args = self._store(args, path + "<arg>", live_out=None)
            try:
                value = live()
            except Exception as e:      # noqa: BLE001 -- the reference's exception is part of its behaviour
                self.log.append((op, path, stored_args, ("raise", type(e).__name__, str(e))))
                raise
            out = []
            self.log.append((op, path, stored_args, ("value", self._store(value, path, out))))
            return out[0]
        assert self.pos < len(self.log), f"reference access {op} {path} past the end of the recording"
        rop, rpath, rargs, (kind, *res) = self.log[self.pos]
        self.pos += 1
        assert (rop, rpath) == (op, path), f"recorded {rop} {rpath}, the test did {op} {path}"
        assert _same(rargs, self._store(args, path + "<arg>", live_out=None)), f"{op} {path}: arguments differ from the recording"
        if kind == "raise":
            raise getattr(builtins, res[0], RuntimeError)(res[1])
        return self._restore(res[0])

    def _store(self, v, path, live_out):
        """Loggable form of `v`; `live_out` (a list) receives what the test gets back while recording."""
        if isinstance(v, _Proxy):
            return _Handle(v._path)
        if _plain(v):
            if live_out is not None:
                live_out.append(v)
            return v
        if _is_task(v):
            from metaworld_b200.benchmarks import Task
            if live_out is not None:
                live_out.append(v)
            return Task(v.env_name, v.data)
        if type(v).__name__ == "Box" and hasattr(v, "low"):
            if live_out is not None:
                live_out.append(v)
            return Box(v.low, v.high, v.shape, v.dtype)
        if isinstance(v, (list, tuple, dict)):
            items = list(v.items()) if isinstance(v, dict) else list(enumerate(v))
            kids, live = [], []
            for k, x in items:
                sub = [] if live_out is not None else None
                kids.append(self._store(x, f"{path}[{k!r}]", sub))
                if sub is not None:
                    live.append(sub[0])
            if live_out is not None:
                live_out.append(dict(zip(v.keys(), live)) if isinstance(v, dict) else type(v)(live) if isinstance(v, list) else tuple(live))
            return dict(zip(v.keys(), kids)) if isinstance(v, dict) else (kids if isinstance(v, list) else tuple(kids))
        if isinstance(v, np.ndarray):      # object array holding reference objects
            if live_out is not None:
                live_out.append(v)
            return np.array([self._store(x, f"{path}[{i}]", None) for i, x in enumerate(v.flat)], dtype=object).reshape(v.shape)
        if live_out is not None:
            live_out.append(_Proxy(self, path, v))
        return _Handle(path)

    def _restore(self, v):
        if isinstance(v, _Handle):
            return _Proxy(self, v.path, None)
        if isinstance(v, dict):
            return {k: self._restore(x) for k, x in v.items()}
        if isinstance(v, (list, tuple)):
            return type(v)(self._restore(x) for x in v)
        return v


@pytest.fixture
def ref(request):
    s = RefSession(request.node.name.replace("[", "_").rstrip("]"))
    yield s
    s.close()


@pytest.fixture
def gym(ref):
    return ref.module("gymnasium")


@pytest.fixture
def metaworld(ref, gym):
    return ref.module("metaworld")


class _Proxy:
    def __init__(self, session, path, target):
        object.__setattr__(self, "_session", session)
        object.__setattr__(self, "_path", path)
        object.__setattr__(self, "_target", target)

    def __getattr__(self, name):
        if name.startswith("__"):
            raise AttributeError(name)
        return self._session.access("getattr", f"{self._path}.{name}", (), lambda: getattr(self._target, name))

    def __setattr__(self, name, value):
        self._session.access("setattr", f"{self._path}.{name}", (value,), lambda: setattr(self._target, name, value))

    def __call__(self, *args, **kw):
        unwrap = (lambda x: x._target if isinstance(x, _Proxy) else x)
        return self._session.access("call", f"{self._path}()", (args, kw),
                                    lambda: self._target(*[unwrap(a) for a in args], **{k: unwrap(x) for k, x in kw.items()}))

    def __getitem__(self, key):
        return self._session.access("getitem", f"{self._path}[{key!r}]", (), lambda: self._target[key])

    def __iter__(self):
        return iter(self._session.access("iter", f"{self._path}", (), lambda: list(self._target)))

    def __len__(self):
        return self._session.access("len", f"{self._path}", (), lambda: len(self._target))

    def __repr__(self):
        return self._session.access("repr", f"{self._path}", (), lambda: repr(self._target))
