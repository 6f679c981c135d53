"""Minimal tabular logger with the surface the hot path uses (rllab/misc/logger.py:56-78,113-232):
log / prefix / record_tabular / dump_tabular / save_itr_params, snapshot modes all|last|gap|none."""
import datetime
import os
import pickle
import sys
from contextlib import contextmanager

_prefixes = []
_tabular = []
_snapshot_dir = None
_snapshot_mode = "none"
_snapshot_gap = 1
_quiet = False
_last_table = {}


def set_quiet(q=True):
    global _quiet
    _quiet = q


def log(s, with_prefix=True, with_timestamp=True):
    if _quiet:
        return
    out = s
    if with_prefix:
        out = "".join(_prefixes) + out
    if with_timestamp:
        out = "%s | %s" % (datetime.datetime.now().strftime("%Y-%m-%d %H:%M:%S.%f"), out)
    sys.stdout.write(out + "\n")
    sys.stdout.flush()


@contextmanager
def prefix(key):
    _prefixes.append(key)
    try:
        yield
    finally:
        _prefixes.pop()


def record_tabular(key, val):
    """val may be a zero-argument callable: it is resolved at dump_tabular().  The device hot path records its
    statistics that way so that the device->host readback waits at the end of the iteration instead of idling the GPU
    in the middle of it."""
    _tabular.append((str(key), val))


def get_last_table():
    """The key/value table of the most recent dump_tabular (tests and bench read results here)."""
    return dict(_last_table)


def dump_tabular(*args, **kwargs):
    global _last_table
    _tabular[:] = [(k, v() if callable(v) else v) for k, v in _tabular]
    _last_table = dict(_tabular)
    if not _quiet and len(_tabular) > 0:
        w = max(len(k) for k, _ in _tabular)
        for k, v in _tabular:
            log("%s  %s" % (k.ljust(w), v), with_timestamp=False)
    del _tabular[:]


def set_snapshot_dir(d):
    global _snapshot_dir
    _snapshot_dir = d


def set_snapshot_mode(m):
    global _snapshot_mode
    _snapshot_mode = m


def set_snapshot_gap(g):
    global _snapshot_gap
    _snapshot_gap = g


def snapshot_enabled():
    """True when save_itr_params writes a file (callers can skip building a snapshot's host copies otherwise)."""
    return bool(_snapshot_dir) and _snapshot_mode != "none"


def save_itr_params(itr, params):
    """rllab/misc/logger.py:216-232 (pickle instead of joblib.dump; same file names)."""
    if not _snapshot_dir or _snapshot_mode == "none":
        return
    os.makedirs(_snapshot_dir, exist_ok=True)
    if _snapshot_mode == "all":
        name = "itr_%d.pkl" % itr
    elif _snapshot_mode == "last":
        name = "params.pkl"
    elif _snapshot_mode == "gap":
        if itr % _snapshot_gap != 0:
            return
        name = "itr_%d.pkl" % itr
    else:
        raise NotImplementedError(_snapshot_mode)
    with open(os.path.join(_snapshot_dir, name), "wb") as f:
        pickle.dump(params, f)
