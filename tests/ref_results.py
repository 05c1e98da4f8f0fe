"""What the reference (oracle/_ref, compiled from the original x265 sources by oracle/Makefile.ref) returned in the
*_oracle_vs_ref tests, stored under tests/golden/ so that those comparisons also run where oracle/_ref cannot be built.

A test makes one RefResults and passes every value it compares through `same(key, ref_fn, value)`:
  * oracle/_ref built: ref_fn() computes the reference's value, `value` must equal it and its digest must equal the stored one;
  * oracle/_ref absent: the digest of `value` must equal the stored digest of the reference's value.
Reference outputs that a test feeds back into the code under test go through `value(key, ref_fn)` and are stored whole.
Tests with thousands of comparisons (the primitive table) use `getter` / `check` / `finish` instead: every comparison is
exact while oracle/_ref is built, and one digest over all of them, in order, is stored per test.
X265_WRITE_GOLDEN=1, with oracle/_ref built, stores what the reference computes instead of checking it."""
import hashlib
import json
import os

import numpy as np
import pytest

from common import ROOT, load_ref

DIGESTS = os.path.join(ROOT, "tests", "golden", "ref_digests.json")
ARRAYS = os.path.join(ROOT, "tests", "golden", "ref_values.npz")
_store = {}


def _load():
    if not _store:
        _store["digests"] = json.load(open(DIGESTS)) if os.path.exists(DIGESTS) else {}
        _store["values"] = dict(np.load(ARRAYS)) if os.path.exists(ARRAYS) else {}
    return _store


def _save():
    with open(DIGESTS, "w") as f:
        json.dump(_store["digests"], f, indent=0, sort_keys=True)
        f.write("\n")
    np.savez_compressed(ARRAYS, **_store["values"])


def digest(v):
    """Digest of an int, a float, an array or a list / tuple / dict of those.  Integer arrays are digested by value and
    shape, not by element type, so that equal results of differently typed buffers agree."""
    h = hashlib.sha256()

    def feed(x):
        if isinstance(x, dict):
            for k in sorted(x):
                h.update(("{%s" % k).encode())
                feed(x[k])
        elif isinstance(x, np.ndarray):
            h.update(("a%s" % (x.shape,)).encode())
            h.update(np.ascontiguousarray(x.astype(np.int64) if x.dtype.kind in "biu" else x).tobytes())
        elif isinstance(x, (list, tuple)):
            h.update(("[%d" % len(x)).encode())
            for y in x:
                feed(y)
        elif isinstance(x, float):
            h.update(("f%r" % x).encode())
        else:
            h.update(("i%d" % int(x)).encode())
    feed(v)
    return h.hexdigest()[:16]


class RefResults:
    def __init__(self, request, depth, name=None):
        """name: where the results are stored when several tests share them (default: the test's own id)."""
        self.R = load_ref(depth)
        self.test = name or "%s::%s" % (request.node.module.__name__, request.node.name)
        self.write = self.R is not None and os.environ.get("X265_WRITE_GOLDEN") == "1"
        store = _load()
        if self.write:
            store["digests"][self.test] = {}
            for k in [k for k in store["values"] if k.startswith(self.test + "/")]:
                del store["values"][k]
            request.addfinalizer(_save)
        elif self.test not in store["digests"]:
            pytest.fail("no stored reference results for %s in %s" % (self.test, DIGESTS))
        self.digests = store["digests"][self.test]
        self.values = store["values"]
        self._n, self._h = 0, hashlib.sha256()

    def same(self, key, ref_fn, value):
        """Asserts that `value` equals the reference's result `key`."""
        if self.R is None:
            assert digest(value) == self.digests[key], "%s differs from the reference's stored result" % key
            return
        r = ref_fn()
        assert digest(r) == digest(value), (key, r, value)
        if self.write:
            self.digests[key] = digest(r)
        else:
            assert digest(r) == self.digests[key], "the reference's %s differs from %s" % (key, DIGESTS)

    def value(self, key, ref_fn):
        """The reference's result `key` (an array or a sequence of ints), computed or stored."""
        name = self.test + "/" + key
        if self.R is None:
            return self.values[name]
        r = ref_fn()
        if self.write:
            self.values[name] = np.asarray(r)
        else:
            assert np.array_equal(np.asarray(r), self.values[name]), "the reference's %s differs from %s" % (key, ARRAYS)
        return r

    def getter(self, make):
        """A table getter (name, restype, argtypes, i, j, k) -> callable or None: the reference's, from `make`, while
        oracle/_ref is built; otherwise a stand-in that does nothing, returned exactly where the reference has the entry."""
        def get(name, restype, argtypes, i=0, j=0, k=0):
            key = "absent %s %d %d %d" % (name, i, j, k)
            if self.R is None:
                return None if key in self.digests else _StandIn()
            f = make(name, restype, argtypes, i, j, k)
            if self.write:
                if f is None:
                    self.digests[key] = "-"
            else:
                assert (f is None) == (key in self.digests), "the reference's table entry %s differs from %s" % (key[7:], DIGESTS)
            return f
        return get

    def check(self, ref_value, value, what=None):
        """One comparison of a sequence: `value` must equal `ref_value` (ignored when oracle/_ref is absent)."""
        if self.R is not None:
            assert digest(ref_value) == digest(value), (what, ref_value, value)
        self._n += 1
        self._h.update(digest(value).encode())

    def finish(self):
        """Compares the digest of every `check` of the test with the reference's stored one."""
        v = (self._n, int(self._h.hexdigest()[:15], 16))
        self.same("checks", lambda: v, v)


class _StandIn:
    def __call__(self, *a):
        return 0
