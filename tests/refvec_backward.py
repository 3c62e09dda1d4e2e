"""Stored outputs of the reference's Chamfer and approximate-EMD backward kernels (tests/golden/ref_metrics_backward.npz).

The same scheme as tests/refvec.py, kept in a file of its own and smaller: outputs of at most refvec.FULL_MAX elements
are stored whole; larger ones as the SHA-256 digest of their bytes, their max-abs value and root-mean-square, and every
SAMPLE_STRIDE-th element of refvec's seeded sample.  The sample positions follow from the tensor's size alone, so they
are not stored.

To record them again (on a GPU, with the reference binaries that `python oracle/build_ref.py` builds into oracle/_ref/):

    LION_REF_RECORD_BACKWARD=tests/golden/ref_metrics_backward.npz python -m pytest tests/test_metrics_backward_gpu.py

In that mode `fn()` runs the reference, the tests compare against its fresh outputs, and the file is written at exit.
"""
import atexit
import os

import numpy as np

from tests import refvec as R

PATH = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ref_metrics_backward.npz")
RECORD = os.environ.get("LION_REF_RECORD_BACKWARD")
SAMPLE_STRIDE = 4

_store = None
_new = {}


def sample_idx(size):
    return R._sample_idx(size)[::SAMPLE_STRIDE]


def record(t):
    a = R._np(t)
    d = {"shape": np.array(a.shape, dtype=np.int64), "dtype": np.array(a.dtype.str)}
    a64 = a.astype(np.float64).ravel()
    d["amax"] = np.array(np.abs(a64).max() if a64.size else 0.0)
    d["rms"] = np.array(np.sqrt(np.mean(a64 * a64)) if a64.size else 0.0)
    if a.size <= R.FULL_MAX:
        d["full"] = a
    else:
        d["digest"] = R._digest(a)
        d["vals"] = a.ravel()[sample_idx(a.size)]
    return d


def _load():
    global _store
    if _store is None:
        _store = dict(np.load(PATH)) if os.path.exists(PATH) and not RECORD else {}
    return _store


def ref_out(key, fn):
    """The reference's outputs for this key, a tuple of refvec.Stored (usable with refvec.equal / close / rms)."""
    if RECORD:
        out = fn()
        for i, t in enumerate(out if isinstance(out, (tuple, list)) else (out,)):
            for k, v in record(t).items():
                _new["%s/%d/%s" % (key, i, k)] = v
    src = _new if RECORD else _load()
    n = sum(1 for k in src if k.startswith(key + "/") and k.endswith("/shape"))
    assert n > 0, "no stored reference output for %r in %s" % (key, PATH)
    res = []
    for i in range(n):
        p = "%s/%d/" % (key, i)
        d = {k[len(p):]: v for k, v in src.items() if k.startswith(p)}
        if "full" not in d:
            d["idx"] = sample_idx(int(np.prod(d["shape"])))
        res.append(R.Stored(d))
    return tuple(res)


def _save():
    if RECORD and _new:
        merged = dict(np.load(RECORD)) if os.path.exists(RECORD) else {}
        merged.update(_new)
        np.savez_compressed(RECORD, **merged)


atexit.register(_save)
