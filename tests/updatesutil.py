"""The update batch on the host build (tests/host_sim/updates_host.cpp), and fabgpu_block_updates' records in updates_oracle's form."""
import ctypes
import os
import subprocess
import tempfile

import numpy as np

from util import ROOT
from blockutil import _p
import mvccutil
import updates_oracle as uo

CC = "mycc"

WORDS = 14
_LIB = None


def lib():
    """built into a temporary directory: the source tree is not written"""
    global _LIB
    if _LIB is None:
        so = os.path.join(tempfile.mkdtemp(prefix="fabgpu_upd_"), "libupdates_host.so")
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-o", so, os.path.join(ROOT, "tests", "host_sim", "updates_host.cpp")])
        L = ctypes.CDLL(so)
        L.hs_new.restype = ctypes.c_void_p
        L.hs_new.argtypes = [ctypes.c_ulonglong]
        L.hs_free.argtypes = [ctypes.c_void_p]
        L.hs_apply.restype = ctypes.c_char_p
        L.hs_apply.argtypes = [ctypes.c_void_p, ctypes.c_int] + [ctypes.c_void_p] * 7 + [ctypes.c_size_t, ctypes.c_ulonglong, ctypes.c_size_t,
                                                                                           ctypes.c_ulonglong, ctypes.POINTER(ctypes.c_int)]
        L.hs_info.argtypes = [ctypes.c_void_p, ctypes.c_void_p]
        L.hs_updates.restype = ctypes.c_char_p
        L.hs_updates.argtypes = [ctypes.c_void_p] + [ctypes.c_void_p] * 3 + [ctypes.c_ulonglong] + [ctypes.c_void_p] * 2 + [ctypes.c_size_t, ctypes.c_void_p,
                                 ctypes.c_size_t, ctypes.c_void_p, ctypes.c_size_t, ctypes.c_void_p, ctypes.POINTER(ctypes.c_int)]
        L.hs_lookup.argtypes = [ctypes.c_void_p, ctypes.c_char_p, ctypes.c_uint32, ctypes.c_char_p, ctypes.c_uint32, ctypes.c_char_p, ctypes.c_uint32,
                                ctypes.c_void_p]
        _LIB = L
    return _LIB


def block_of(txs):
    """the transactions' read/write sets (updates_oracle.encode) back to back: (blob, results pairs, htype)"""
    blob, res, ht = b"", [], []
    for tx in txs:
        if tx is None:
            res += [0, 0]; ht.append(1)
            continue
        rw = uo.encode(tx)
        res += [len(blob) + 8, len(rw)]; ht.append(3)
        blob += bytes(8) + rw
    return np.frombuffer(blob + bytes(64), np.uint8).copy(), np.array(res or [0], np.uint32), np.array(ht or [0], np.uint8)


def decode(words, meta, src):
    """records (WORDS uint32 each) with their bytes read from the submitted block `src` and the metadata buffer -> updates_oracle records"""
    src, meta = bytes(src), bytes(meta)
    out = []
    for w in np.asarray(words, np.uint32).reshape(-1, WORDS).tolist():
        tx, op, vs, ms = w[:4]
        seg = lambda o, n: src[o:o + n]
        value = None if vs == 0 else seg(w[10], w[11]) if vs == 1 else uo.COMMITTED
        md = None if ms == 0 else meta[w[12]:w[12] + w[13]] if ms == 1 else uo.COMMITTED
        out.append((tx, "put" if op == 1 else "del", seg(w[4], w[5]).decode(), seg(w[6], w[7]).decode(), seg(w[8], w[9]), value, md))
    return out


class HostUpdates(mvccutil.HostState):
    def __init__(self, seed=0x5EED):
        self.L = lib()
        self.h = ctypes.c_void_p(self.L.hs_new(seed))
        self.max_bytes = 0

    def updates(self, block_num, txs, tv, rec_cap=4096, meta_cap=1 << 16):
        """(flags, records or None when incomplete, full counts)"""
        blob, res, ht = block_of(txs)
        tv = np.ascontiguousarray(np.asarray(list(tv) or [0], np.uint8))
        flags = np.zeros(max(len(txs), 1), np.uint8)
        rec = np.zeros(max(rec_cap, 1) * WORDS, np.uint32)
        meta = np.zeros(max(meta_cap, 1), np.uint8)
        n = (ctypes.c_size_t * 2)()
        complete = ctypes.c_int(0)
        err = self.L.hs_updates(self.h, _p(blob), _p(res), _p(ht), block_num, _p(tv), _p(flags), len(txs), _p(rec), rec_cap, _p(meta), meta_cap, n,
                                ctypes.byref(complete))
        if err is not None:
            raise mvccutil.StateError(err.decode(), False)
        recs = decode(rec[:min(n[0], rec_cap) * WORDS], meta[:min(n[1], meta_cap)], blob) if complete.value else None
        return flags[:len(txs)].tolist(), recs, (int(n[0]), int(n[1]))


def random_tx(rng, pool, t):
    """mvccutil.random_tx's shape with distinct values and metadata entries: reads, upserts, deletes, metadata writes with and without
    entries (now and then a second write of a key), a hashed write and hashed metadata write"""
    ns = dict(ns=CC, reads=[], writes=[], md=[], colls=[])
    for _ in range(rng.integers(0, 3)):
        k = pool[rng.integers(len(pool))]
        ns["reads"].append((k, None if rng.random() < 0.3 else (int(rng.integers(0, 3)), int(rng.integers(0, 3)))))
    for j in range(rng.integers(1, 4)):
        k = pool[rng.integers(len(pool))]
        x = rng.random()
        if x < 0.2:
            ns["md"].append((k, None if rng.random() < 0.3 else [("VALIDATION_PARAMETER", b"p%d.%d" % (t, j))] + ([("x", b"")] if x < 0.05 else [])))
        else:
            ns["writes"].append((k, uo.DEL if x < 0.35 else b"v%d.%d" % (t, j)))
    if rng.random() < 0.2:
        hk = b"h" + pool[rng.integers(len(pool))].encode()
        ns["colls"].append(("c", [], [(hk, b"hv%d" % t)], [(hk, [("VALIDATION_PARAMETER", b"hp%d" % t)])] if rng.random() < 0.5 else []))
    return [ns]
