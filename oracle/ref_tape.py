"""TEST INFRASTRUCTURE: record / replay of what the reference returns to a test.

A test that compares the product with the live reference reaches the reference only through
`ref_harness.load_reference_foundation()`.  Under `taped` that call returns a proxy.  With a reference checkout present
the proxy forwards every operation (attribute, call, item, `in`, `len`, iteration) to the real object and records each
plain-data result (numbers, strings, numpy arrays and containers of them), each exception, and the fact that a result was
an object (which is wrapped again).  Without a checkout the same operations are answered from the recording under
tests/golden/reference_tapes/, so the comparison runs unchanged.  Every operation is recorded with its kind, name and a
digest of its plain-data arguments: a test that asks the reference anything else, or passes it different actions than
when the tape was recorded, fails with the position of the first difference.

With a reference checkout, `AIE_RECORD_REFERENCE_TAPES=1 python -m pytest -m reference tests` (re)writes every tape.
"""
import functools
import hashlib
import lzma
import os
import pickle
import re

import numpy as np

TAPE_DIR = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden", "reference_tapes")
_LEAF = (np.ndarray, np.generic, int, float, complex, bool, str, bytes, type(None), range, slice)
_VIEWS = (type({}.keys()), type({}.values()), type({}.items()))

_active = None   # the tape of the running test
_MAX_TWISTS = 20000   # an MT19937 key is stored as "the previous key, twisted k times" when k is at most this


def _is_leaf(v):
    if isinstance(v, np.ndarray):
        return v.dtype != object
    if isinstance(v, _LEAF):
        return True
    if isinstance(v, (list, tuple)):
        return all(_is_leaf(x) for x in v)
    if isinstance(v, dict):
        return all(_is_leaf(k) and _is_leaf(x) for k, x in v.items())
    return False


def _unwrap(v):
    if isinstance(v, _Proxy):
        return object.__getattribute__(v, "_o")
    if isinstance(v, (list, tuple)):
        return type(v)(_unwrap(x) for x in v)
    if isinstance(v, dict):
        return {k: _unwrap(x) for k, x in v.items()}
    return v


def _digest(v):
    """Digest of the plain data in a call's arguments (objects of the reference count only by their place)."""
    def norm(x):
        if isinstance(x, _Proxy):
            return "<ref>"
        if isinstance(x, (list, tuple)):
            return [norm(y) for y in x]
        if isinstance(x, dict):
            return sorted((repr(k), norm(y)) for k, y in x.items())
        if isinstance(x, np.ndarray):
            return (str(x.dtype), x.shape, x.tobytes())
        if isinstance(x, np.generic):
            return x.item()
        return x if isinstance(x, _LEAF) else "<%s>" % type(x).__name__
    return hashlib.sha1(pickle.dumps(norm(v), protocol=4)).hexdigest()[:12]


def _twist(key):
    rs = np.random.RandomState()
    rs.set_state(("MT19937", key, 624))
    rs.bytes(4 * 624)   # 624 32-bit words: exactly one twist
    return rs.get_state()[1]


class Tape:
    def __init__(self, name, record):
        self.name, self.record, self.pos = name, record, 0
        self.mt = None   # the last MT19937 key seen in this tape
        self.path = os.path.join(TAPE_DIR, re.sub(r"[^A-Za-z0-9_.\[\]-]+", "_", name) + ".pkl.xz")
        if record:
            self.events = []
        else:
            if not os.path.exists(self.path):
                raise AssertionError("no reference checkout and no recorded tape %s" % os.path.relpath(self.path))
            with lzma.open(self.path, "rb") as f:
                self.events = pickle.load(f)

    def save(self):
        os.makedirs(TAPE_DIR, exist_ok=True)
        with lzma.open(self.path, "wb", preset=9) as f:
            pickle.dump(self.events, f, protocol=4)

    def _next(self, key):
        if self.pos >= len(self.events):
            raise AssertionError("%s: the test asks the reference more than was recorded (%r)" % (self.name, key))
        ev = self.events[self.pos]
        self.pos += 1
        if ev[0] != key:
            raise AssertionError("%s: operation %d on the reference differs from the recording: %r, recorded %r"
                                 % (self.name, self.pos - 1, key, ev[0]))
        return ev

    def _mt_code(self, v):
        """MT19937 keys (uint32 [624]) are random data: each one is coded as the number of twists from the previous one."""
        if isinstance(v, np.ndarray) and v.dtype == np.uint32 and v.shape == (624,):
            prev, self.mt = self.mt, v.copy()
            if prev is not None:
                for k in range(_MAX_TWISTS + 1):
                    if np.array_equal(prev, v):
                        return ("MT19937 twists", k)
                    prev = _twist(prev)
            return v
        if isinstance(v, (list, tuple)):
            return type(v)(self._mt_code(x) for x in v)
        if isinstance(v, dict):
            return {k: self._mt_code(x) for k, x in v.items()}
        return v

    def _mt_decode(self, v):
        if isinstance(v, tuple) and len(v) == 2 and v[0] == "MT19937 twists":
            key = self.mt
            for _ in range(v[1]):
                key = _twist(key)
            self.mt = key.copy()
            return key
        if isinstance(v, np.ndarray) and v.dtype == np.uint32 and v.shape == (624,):
            self.mt = v.copy()
            return v
        if isinstance(v, (list, tuple)):
            return type(v)(self._mt_decode(x) for x in v)
        if isinstance(v, dict):
            return {k: self._mt_decode(x) for k, x in v.items()}
        return v

    def _wrap(self, key, v):
        """Record (or replay) one result: plain data as it is, sequences of objects element by element, objects as proxies."""
        if self.record:
            if isinstance(v, _VIEWS):
                v = list(v)
            if _is_leaf(v):
                self.events.append((key, "L", pickle.dumps(self._mt_code(v), protocol=4)))
                return v
            if isinstance(v, (list, tuple)):
                self.events.append((key, "S", len(v), type(v) is tuple))
                seq = [self._wrap(key + ("#%d" % i,), x) for i, x in enumerate(v)]
                return tuple(seq) if isinstance(v, tuple) else seq
            self.events.append((key, "O"))
            return _Proxy(self, v)
        ev = self._next(key)
        if ev[1] == "L":
            return self._mt_decode(pickle.loads(ev[2]))
        if ev[1] == "S":
            seq = [self._wrap(key + ("#%d" % i,), None) for i in range(ev[2])]
            return tuple(seq) if ev[3] else seq
        if ev[1] == "E":
            raise pickle.loads(ev[2])
        return _Proxy(self, None)

    def op(self, key, fn):
        if not self.record:
            return self._wrap(key, None)
        try:
            v = fn()
        except Exception as ex:
            try:
                blob = pickle.dumps(ex, protocol=4)
                pickle.loads(blob)
            except Exception:
                blob = pickle.dumps(RuntimeError("%s: %s" % (type(ex).__name__, ex)), protocol=4)
            self.events.append((key, "E", blob))
            raise
        return self._wrap(key, v)


class _Proxy:
    __slots__ = ("_t", "_o")

    def __init__(self, tape, obj):
        object.__setattr__(self, "_t", tape)
        object.__setattr__(self, "_o", obj)

    def __getattr__(self, name):
        o = object.__getattribute__(self, "_o")
        return object.__getattribute__(self, "_t").op(("getattr", name), lambda: getattr(o, name))

    def __setattr__(self, name, value):
        o = object.__getattribute__(self, "_o")
        object.__getattribute__(self, "_t").op(("setattr", name, _digest(value)), lambda: setattr(o, name, _unwrap(value)))

    def __call__(self, *a, **k):
        o = object.__getattribute__(self, "_o")
        return object.__getattribute__(self, "_t").op(("call", _digest((a, k))), lambda: o(*_unwrap(a), **_unwrap(k)))

    def __getitem__(self, i):
        o = object.__getattribute__(self, "_o")
        return object.__getattribute__(self, "_t").op(("getitem", _digest(i)), lambda: o[_unwrap(i)])

    def __contains__(self, x):
        o = object.__getattribute__(self, "_o")
        return object.__getattribute__(self, "_t").op(("contains", _digest(x)), lambda: _unwrap(x) in o)

    def __len__(self):
        o = object.__getattribute__(self, "_o")
        return object.__getattribute__(self, "_t").op(("len",), lambda: len(o))

    def __iter__(self):
        o = object.__getattribute__(self, "_o")
        return iter(object.__getattribute__(self, "_t").op(("iter",), lambda: list(o)))

    def __bool__(self):
        o = object.__getattribute__(self, "_o")
        return object.__getattribute__(self, "_t").op(("bool",), lambda: bool(o))


def active():
    return _active


def recorded(fn):
    """For the harness's converters (reference env -> plain arrays): while a tape runs, the call is one recorded operation
    (its result, not the many attribute reads it makes); outside a tape it is the plain function."""
    @functools.wraps(fn)
    def run(*a, **k):
        global _active
        t = _active
        if t is None:
            return fn(*a, **k)
        if not t.record:
            return t.op(("fn", fn.__name__, _digest((a, k))), None)

        def live():
            global _active
            _active = None   # the converter reads the real objects directly
            try:
                return fn(*_unwrap(a), **_unwrap(k))
            finally:
                _active = t
        return t.op(("fn", fn.__name__, _digest((a, k))), live)
    return run


def global_stream_state():
    """np.random.get_state() of the global stream the reference draws from (recorded like any other reference result)."""
    if _active is None:
        return np.random.get_state()
    return _active.op(("np.random.get_state",), np.random.get_state)


def wrap_foundation(foundation):
    """What load_reference_foundation() hands out while a tape runs (foundation is None when replaying)."""
    return _Proxy(_active, foundation)


def taped(fn):
    """Run a test against its reference tape: live and recording with a reference checkout, replayed without one."""
    from oracle import ref_harness as rh

    @functools.wraps(fn)
    def run(*a, **k):
        global _active
        node = os.environ["PYTEST_CURRENT_TEST"].rsplit(" ", 1)[0]
        name = node.split("/")[-1].replace(".py::", "__")
        _active = Tape(name, record=rh.reference_available())
        try:
            return fn(*a, **k)
        finally:
            t, _active = _active, None
            if t.record and os.environ.get("AIE_RECORD_REFERENCE_TAPES", "0") not in ("", "0"):
                t.save()
    return run
