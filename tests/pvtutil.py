"""The private-data check on the host build (tests/host_sim/pvt_host.cpp): the same pvtdata.cuh steps the library launches, one item at
a time, over public read/write sets back to back."""
import ctypes
import os
import subprocess
import tempfile

import numpy as np

from util import ROOT
from blockutil import _blob, _p

_LIB = None


def lib():
    """built into a temporary directory: the source tree is not written"""
    global _LIB
    if _LIB is None:
        so = os.path.join(tempfile.mkdtemp(prefix="fabgpu_pvt_"), "libpvt_host.so")
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-o", so, os.path.join(ROOT, "tests", "host_sim", "pvt_host.cpp")])
        L = ctypes.CDLL(so)
        L.pv_host.restype = None
        L.pv_host.argtypes = [ctypes.c_void_p] * 3 + [ctypes.c_size_t] + [ctypes.c_void_p] * 4 + [ctypes.c_size_t, ctypes.c_void_p, ctypes.c_void_p]
        _LIB = L
    return _LIB


def block_of(rwsets):
    """public TxReadWriteSet bytes (None: a non-endorser transaction) back to back: (blob, results pairs, htype)"""
    blob, res, ht = b"", [], []
    for rw in rwsets:
        if rw is None:
            res += [0, 0]; ht.append(1)
            continue
        res += [len(blob) + 8, len(rw)]; ht.append(3)
        blob += bytes(8) + rw
    return np.frombuffer(blob + bytes(64), np.uint8).copy(), np.array(res or [0], np.uint32), np.array(ht or [0], np.uint8)


def host_check(rwsets, flags, pvt):
    """-> ((code, seq, ns, coll), {seq: (code, ns, coll)}) as fabgpu_validate_pvtdata returns them"""
    blob, res, ht = block_of(rwsets)
    fl = np.array(list(flags) or [0], np.uint8)
    seqs = sorted(pvt)
    pb_, off = _blob([pvt[s] for s in seqs])
    sq = np.array(seqs or [0], np.uint32)
    st = np.zeros(3 * max(len(seqs), 1), np.int32)
    out = np.zeros(4, np.int32)
    lib().pv_host(_p(blob), _p(res), _p(ht), len(rwsets), _p(fl), _p(pb_), _p(off), _p(sq), len(seqs), _p(st), _p(out))
    return tuple(int(x) for x in out), {s: tuple(int(x) for x in st[3 * i:3 * i + 3]) for i, s in enumerate(seqs)}
