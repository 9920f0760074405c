"""The world-state version table and the MVCC stage on the host build (tests/host_sim/mvcc_host.cpp), and the state's array form for
fabgpu_state_versions / _update."""
import ctypes
import os
import subprocess
import tempfile

import numpy as np

from util import ROOT
from blockutil import _blob, _p
import mvcc_oracle as mo

_LIB = None


def lib():
    """built into a temporary directory: the source tree is not written"""
    global _LIB
    if _LIB is None:
        so = os.path.join(tempfile.mkdtemp(prefix="fabgpu_mvcc_"), "libmvcc_host.so")
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-o", so, os.path.join(ROOT, "tests", "host_sim", "mvcc_host.cpp")])
        L = ctypes.CDLL(so)
        L.hs_new.restype = ctypes.c_void_p
        L.hs_new.argtypes = [ctypes.c_ulonglong]
        L.hs_free.argtypes = [ctypes.c_void_p]
        L.hs_apply.restype = ctypes.c_char_p
        L.hs_apply.argtypes = [ctypes.c_void_p, ctypes.c_int] + [ctypes.c_void_p] * 7 + [ctypes.c_size_t, ctypes.c_ulonglong, ctypes.c_size_t,
                                                                                           ctypes.c_ulonglong, ctypes.POINTER(ctypes.c_int)]
        L.hs_info.argtypes = [ctypes.c_void_p, ctypes.c_void_p]
        L.hs_mvcc.restype = ctypes.c_char_p
        L.hs_mvcc.argtypes = [ctypes.c_void_p] + [ctypes.c_void_p] * 3 + [ctypes.c_ulonglong, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_size_t,
                                                                         ctypes.c_ulonglong, ctypes.POINTER(ctypes.c_int)]
        L.hs_lookup.argtypes = [ctypes.c_void_p, ctypes.c_char_p, ctypes.c_uint32, ctypes.c_char_p, ctypes.c_uint32, ctypes.c_char_p, ctypes.c_uint32,
                                ctypes.c_void_p]
        _LIB = L
    return _LIB


def arrays(entries):
    """[((ns, coll, key), version or mvcc_oracle.REMOVE)] -> (ns_blob, ns_off, coll_blob, coll_off, key_blob, key_off, ver)"""
    nb, no = _blob([k[0].encode() for k, _ in entries])
    cb, co = _blob([k[1].encode() for k, _ in entries])
    kb, ko = _blob([bytes(k[2]) for k, _ in entries])
    ver = np.array([x for _, v in entries for x in v] or [0], np.uint64)
    return nb, no, cb, co, kb, ko, ver


def state_entries(state):
    """a state dict's installable entries (keys the oracle marks unknown are left out: the table learns those from blocks)"""
    return [(k, v) for k, v in sorted(state.items()) if v != mo.UNKNOWN]


def block_of(txs):
    """The transactions' read/write sets back to back (the host stage reads only ChaincodeAction.results): (blob, results pairs, htype)"""
    blob, res, ht = b"", [], []
    for tx in txs:
        if tx is None:
            res += [0, 0]; ht.append(1)
            continue
        rw = mo.encode(tx)
        res += [len(blob) + 8, len(rw)]; ht.append(3)
        blob += bytes(8) + rw
    return np.frombuffer(blob + bytes(64), np.uint8).copy(), np.array(res or [0], np.uint32), np.array(ht or [0], np.uint8)


class StateError(ValueError):
    def __init__(self, msg, failed):
        super().__init__(msg)
        self.failed = failed


class HostState:
    def __init__(self, seed=0x5EED, max_bytes=0):
        self.L = lib()
        self.h = ctypes.c_void_p(self.L.hs_new(seed))
        self.max_bytes = max_bytes

    def _apply(self, replace, entries, height, hint):
        a = arrays(entries)
        failed = ctypes.c_int(0)
        err = self.L.hs_apply(self.h, int(replace), *[_p(x) for x in a], len(entries), height, hint, self.max_bytes, ctypes.byref(failed))
        if err is not None:
            raise StateError(err.decode(), bool(failed.value))

    def replace(self, entries, height, hint=0):
        self._apply(True, entries, height, hint)

    def update(self, entries, height):
        self._apply(False, entries, height, 0)

    def info(self):
        out = (ctypes.c_ulonglong * 4)()
        self.L.hs_info(self.h, out)
        return tuple(int(x) for x in out)

    def mvcc(self, block_num, txs, tv):
        blob, res, ht = block_of(txs)
        tv = np.ascontiguousarray(np.asarray(tv, np.uint8))
        flags = np.zeros(max(len(txs), 1), np.uint8)
        failed = ctypes.c_int(0)
        err = self.L.hs_mvcc(self.h, _p(blob), _p(res), _p(ht), block_num, _p(tv if tv.size else np.zeros(1, np.uint8)), _p(flags), len(txs),
                             self.max_bytes, ctypes.byref(failed))
        if err is not None:
            raise StateError(err.decode(), bool(failed.value))
        return flags[:len(txs)].tolist()

    def lookup(self, key):
        ver = (ctypes.c_ulonglong * 2)()
        st = self.L.hs_lookup(self.h, key[0].encode(), len(key[0].encode()), key[1].encode(), len(key[1].encode()), bytes(key[2]), len(key[2]), ver)
        return st, (int(ver[0]), int(ver[1]))

    def __del__(self):
        try:
            self.L.hs_free(self.h)
        except Exception:
            pass


def random_tx(rng, pool, ns_name="mycc", unreached=0.01):
    """a random transaction over a key pool: reads with random versions, writes (now and then without a value, or of one key twice),
    deletes, metadata writes (with and without entries), a hashed read and write,
    now and then a range query, and (with probability `unreached`) one whose write set cannot be enumerated"""
    ns = dict(ns=ns_name, reads=[], writes=[], md=[], colls=[])
    for _ in range(rng.integers(0, 3)):
        k = pool[rng.integers(len(pool))]
        ns["reads"].append((k, None if rng.random() < 0.3 else (int(rng.integers(0, 3)), int(rng.integers(0, 3)))))
    for _ in range(rng.integers(0, 3)):
        k = pool[rng.integers(len(pool))]
        x = rng.random()
        if x < 0.15:
            ns["md"].append(k if rng.random() < 0.7 else (k, False))
        else:
            ns["writes"].append((k, x < 0.3, rng.random() < 0.95))
    if rng.random() < 0.2:
        ns["colls"].append(("c", [(b"h" + pool[rng.integers(len(pool))].encode(), None)], [(b"h" + pool[rng.integers(len(pool))].encode(), False)], []))
    if rng.random() < 0.03:
        ns["range"] = True
    return None if rng.random() < unreached else [ns]
