"""The MVCC stage with an ordered key index on the host build (tests/host_sim/range_host.cpp), and running range cases against
range_oracle."""
import ctypes
import os
import subprocess
import tempfile

import numpy as np

from util import ROOT
from blockutil import _p
import mvccutil
import range_oracle as ro

_LIB = None


def lib():
    """built into a temporary directory: the source tree is not written"""
    global _LIB
    if _LIB is None:
        so = os.path.join(tempfile.mkdtemp(prefix="fabgpu_range_"), "librange_host.so")
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-o", so, os.path.join(ROOT, "tests", "host_sim", "range_host.cpp")])
        L = ctypes.CDLL(so)
        L.rh_new.restype = ctypes.c_void_p
        L.rh_new.argtypes = [ctypes.c_ulonglong]
        L.rh_free.argtypes = [ctypes.c_void_p]
        L.rh_apply.restype = ctypes.c_char_p
        L.rh_apply.argtypes = [ctypes.c_void_p, ctypes.c_int] + [ctypes.c_void_p] * 7 + [ctypes.c_size_t, ctypes.c_ulonglong, ctypes.c_size_t,
                                                                                           ctypes.c_ulonglong, ctypes.POINTER(ctypes.c_int)]
        L.rh_info.argtypes = [ctypes.c_void_p, ctypes.c_void_p]
        L.rh_index_info.argtypes = [ctypes.c_void_p, ctypes.c_void_p]
        L.rh_mvcc.restype = ctypes.c_char_p
        L.rh_mvcc.argtypes = [ctypes.c_void_p] + [ctypes.c_void_p] * 3 + [ctypes.c_ulonglong, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_size_t,
                                                                         ctypes.c_ulonglong, ctypes.POINTER(ctypes.c_int)]
        L.rh_lookup.argtypes = [ctypes.c_void_p, ctypes.c_char_p, ctypes.c_uint32, ctypes.c_char_p, ctypes.c_uint32, ctypes.c_char_p, ctypes.c_uint32,
                                ctypes.c_void_p]
        _LIB = L
    return _LIB


def block_of(txs):
    """as mvccutil.block_of, with range_oracle's encoding"""
    blob, res, ht = b"", [], []
    for tx in txs:
        if tx is None:
            res += [0, 0]; ht.append(1)
            continue
        rw = ro.encode(tx)
        res += [len(blob) + 8, len(rw)]; ht.append(3)
        blob += bytes(8) + rw
    return np.frombuffer(blob + bytes(64), np.uint8).copy(), np.array(res or [0], np.uint32), np.array(ht or [0], np.uint8)


class RangeHost:
    def __init__(self, seed=0x5EED):
        self.L = lib()
        self.h = ctypes.c_void_p(self.L.rh_new(seed))

    def _apply(self, mode, entries, height, hint=0):
        a = mvccutil.arrays(entries)
        failed = ctypes.c_int(0)
        err = self.L.rh_apply(self.h, mode, *[_p(x) for x in a], len(entries), height, hint, 0, ctypes.byref(failed))
        if err is not None:
            raise mvccutil.StateError(err.decode(), bool(failed.value))

    def replace(self, entries, height, indexed=True):
        self._apply(2 if indexed else 1, entries, height)

    def update(self, entries, height):
        self._apply(0, entries, height)

    def info(self):
        out = (ctypes.c_ulonglong * 4)()
        self.L.rh_info(self.h, out)
        return tuple(int(x) for x in out)

    def index_info(self):
        out = (ctypes.c_ulonglong * 3)()
        self.L.rh_index_info(self.h, out)
        return tuple(int(x) for x in out)

    def mvcc(self, block_num, txs, tv):
        blob, res, ht = block_of(txs)
        tv = np.ascontiguousarray(np.asarray(tv, np.uint8))
        flags = np.zeros(max(len(txs), 1), np.uint8)
        failed = ctypes.c_int(0)
        err = self.L.rh_mvcc(self.h, _p(blob), _p(res), _p(ht), block_num, _p(tv if tv.size else np.zeros(1, np.uint8)), _p(flags), len(txs), 0,
                             ctypes.byref(failed))
        if err is not None:
            raise mvccutil.StateError(err.decode(), bool(failed.value))
        return flags[:len(txs)].tolist()

    def lookup(self, key):
        ver = (ctypes.c_ulonglong * 2)()
        st = self.L.rh_lookup(self.h, key[0].encode(), len(key[0].encode()), key[1].encode(), len(key[1].encode()), bytes(key[2]), len(key[2]), ver)
        return st, (int(ver[0]), int(ver[1]))

    def __del__(self):
        try:
            self.L.rh_free(self.h)
        except Exception:
            pass


def run_case(state0, steps, mvcc, update):
    """Runs a case's steps from height 1: a block (txs, tv, codes) through mvcc(block_num, txs, tv) -> flags and the oracle, or
    ("update", entries) through update(entries, height) and the oracle's state.  Closes open blocks as a peer would.  Returns
    [(got, oracle flags, codes)] per block and the oracle's final state."""
    state = dict(state0)
    height = 1
    out = []
    for step in steps:
        if step[0] == "update":
            update(step[1], height)
            for k, v in step[1]:
                if v == mvccutil.mo.REMOVE:
                    state.pop(k, None)
                else:
                    state[k] = v
            continue
        txs, tv, codes = step
        got = mvcc(height, txs, tv)
        exp, state, is_open = ro.validate(state, height, txs, tv)
        out.append((got, exp, codes))
        if is_open:
            update([], height + 1)
        height += 1
    return out, state


def random_range_tx(rng, pool, state=None, ns_name="mycc", p_range=0.5):
    """mvccutil.random_tx with, now and then, a range query over the pool: its reads are the committed results of the range in `state`
    (right unless the block's earlier writes or a perturbation change them), as raw reads or, now and then, a Merkle summary of
    max_degree 2 or 3"""
    tx = mvccutil.random_tx(rng, pool, ns_name, unreached=0.005)
    if tx is None:
        return None
    tx[0].pop("range", None)
    if rng.random() < p_range:
        ks = sorted(pool)
        i, j = sorted(int(x) for x in rng.integers(0, len(ks) + 1, 2))
        start, end = ks[i] if i < len(ks) else "zz", ks[j] if j < len(ks) else ""
        exhausted = bool(rng.random() < 0.7)
        try:
            res = list(ro.results(state or {}, {}, 0, ns_name, start, end, exhausted))
        except ro.Undetermined:
            res = [(k.encode(), (0, 0)) for k in ks[i:j]]
        x = rng.random()
        if x < 0.15 and res:
            res = res[:-1]
        elif x < 0.25:
            res = res + [(b"zzz", (0, 1))]
        elif x < 0.35 and res:
            res[0] = (res[0][0], (res[0][1][0], res[0][1][1] + 1))
        if rng.random() < 0.25:
            d = int(rng.integers(2, 4))
            summ = ro.summary_of(res, d) if res else None
            reads = summ if summ is not None else ro.Merkle(d, 1, [])
        else:
            reads = res
        tx[0]["ranges"] = [(start, end, exhausted, reads)]
    return tx
