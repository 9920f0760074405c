"""The device-side block logic run on the host with a committed tx-id set: v13util.device_flags over the host build of
tests/host_sim/blockdev_txid_host.cpp, whose decide stage also takes the set fabgpu_committed_txids / _add would install (the library's
own argument checks, canonical filter, insert, growth and lookup)."""
import ctypes
import hashlib
import os
import subprocess
import tempfile

import numpy as np

from oracle import bccsp_sw as o
from oracle import fast
from util import ROOT, pkg
from blockutil import _blob, _p
import v13util

MODE_V20, MODE_V13 = v13util.MODE_V20, v13util.MODE_V13
_LIB = None


def txid_lib():
    """built into a temporary directory: the source tree is not written"""
    global _LIB
    if _LIB is None:
        d = os.path.join(ROOT, "tests", "host_sim")
        so = os.path.join(tempfile.mkdtemp(prefix="fabgpu_txid_"), "libblockdev_txid_host.so")
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-o", so, os.path.join(d, "blockdev_txid_host.cpp"),
                               os.path.join(ROOT, "fabric-mod_b200", "csrc", "blockval.cpp")])
        L = ctypes.CDLL(so)
        L.bd_new.restype = ctypes.c_void_p
        L.kl_new.restype = ctypes.c_void_p
        L.kl_apply.restype = ctypes.c_char_p
        L.txs_new.restype = ctypes.c_void_p
        L.txs_new.argtypes = [ctypes.c_ulonglong]
        L.txs_apply.restype = ctypes.c_char_p
        L.txs_apply.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_size_t, ctypes.c_size_t,
                                ctypes.c_ulonglong, ctypes.POINTER(ctypes.c_int)]
        L.txs_info.argtypes = [ctypes.c_void_p, ctypes.c_void_p]
        L.txs_lookup.argtypes = [ctypes.c_void_p, ctypes.c_char_p]
        L.txs_max_probe.restype = ctypes.c_ulonglong
        L.txs_max_probe.argtypes = [ctypes.c_void_p]
        L.txs_free.argtypes = [ctypes.c_void_p]
        _LIB = L
    return _LIB


class SetError(ValueError):
    """a call the library refuses (FABGPU_E_ARG) or that breaks the set (failed = True, FABGPU_E_CUDA)"""

    def __init__(self, msg, failed):
        super().__init__(msg)
        self.failed = failed


class HostSet:
    """The committed tx-id set on the host, driven by the library's own code.  max_bytes: FABGPU_TXID_MAX_BYTES (0: no bound)."""

    def __init__(self, seed=0x5EED, max_bytes=0):
        self.L = txid_lib()
        self.h = ctypes.c_void_p(self.L.txs_new(seed))
        self.max_bytes = max_bytes

    def apply(self, replace, ids, kinds=None, capacity=0):
        ids = [x.encode() if isinstance(x, str) else bytes(x) for x in ids]
        b, off = _blob(ids)
        k = None if kinds is None else np.ascontiguousarray(np.asarray(list(kinds) or [0], np.uint8))
        failed = ctypes.c_int(0)
        err = self.L.txs_apply(self.h, int(replace), _p(b), _p(off), None if k is None else _p(k), len(ids), capacity, self.max_bytes, ctypes.byref(failed))
        if err is not None:
            raise SetError(err.decode(), bool(failed.value))

    def info(self):
        out = (ctypes.c_ulonglong * 2)()
        self.L.txs_info(self.h, out)
        return int(out[0]), int(out[1])

    def lookup(self, id32):
        return self.L.txs_lookup(self.h, bytes(id32))

    def max_probe(self):
        return int(self.L.txs_max_probe(self.h))

    def __del__(self):
        try:
            self.L.txs_free(self.h)
        except Exception:
            pass


def device_flags(env_blob, env_off, identities, channel, nodes, principals, mode=MODE_V20, policies=None, versions=None, principal_bits=None,
                 collections=None, key_calls=(), txid_calls=None, writes_hint=32):
    """v13util.device_flags with a committed tx-id set: txid_calls = [(replace, ids, kinds)] applied in order to a fresh set (None: no
    set installed).  mode defaults to v2.0 here."""
    from oracle import goasn1
    L = txid_lib()
    ts = None
    if txid_calls is not None:
        ts = HostSet()
        for replace, ids, kinds in txid_calls:
            ts.apply(replace, ids, kinds)
    nodes = np.ascontiguousarray(nodes, np.int32).reshape(-1, 4)
    kt = v13util._KeyTable.__new__(v13util._KeyTable)
    kt.L, kt.h, kt.base, kt.np = L, ctypes.c_void_p(L.kl_new()), nodes.shape[0], len(principals)
    for replace, kn, table in key_calls:
        kt.apply(replace, kn, table)
    idb, ido = _blob([bytes(i[0]) for i in identities])
    mb, mo = _blob([i[1].encode() for i in identities])
    keys = np.ascontiguousarray(np.frombuffer(b"".join(bytes(i[2]) for i in identities), np.uint8)).reshape(-1, 64)
    valid = np.array([1 if i[3] else 0 for i in identities], np.uint8)
    pbb, pbo = _blob([p.encode() for p in principals])
    h = ctypes.c_void_p(L.bd_new(_p(idb), _p(ido), _p(mb), _p(mo), _p(valid), len(identities), _p(nodes), nodes.shape[0], _p(pbb), _p(pbo),
                                 len(principals), channel.encode()))
    groups = np.ascontiguousarray(pkg().binding.identity_groups(identities), np.int32)
    L.bd_groups(h, _p(groups), len(identities))
    names = sorted(policies) if policies else []
    if names:
        nb, no = _blob([n.encode() for n in names])
        roots = np.array([policies[n] for n in names], np.int32)
        L.bd_namespaces(h, _p(nb), _p(no), _p(roots), len(names))
    vb, vo = _blob([(versions or {}).get(n, "").encode() for n in names])
    blob = np.frombuffer(env_blob, np.uint8) if len(env_blob) else np.zeros(1, np.uint8)
    env_off = np.ascontiguousarray(env_off, np.uint32)
    T = env_off.shape[0] - 1
    n_rec = ctypes.c_uint32(0)
    J = T + L.v13_plan(kt.h, h, _p(blob), _p(env_off), T, writes_hint, mode, ctypes.byref(n_rec))
    ident, gok = ctypes.c_int(0), ctypes.c_int(0)
    r = (ctypes.c_uint8 * 32)(); s = (ctypes.c_uint8 * 32)(); segs = (ctypes.c_uint32 * 12)()
    key_idx, digs, sigs, live = [], [], [], []

    def msg(sg, base=0):
        return b"".join(env_blob[sg[base + k]: sg[base + k] + sg[base + 3 + k]] for k in range(3))
    for j in range(J):
        L.bd_job(h, j, ctypes.byref(ident), ctypes.byref(gok), r, s, segs)
        if ident.value < 0 or not gok.value:
            continue
        live.append(j)
        key_idx.append(ident.value)
        digs.append(hashlib.sha256(msg(segs)).digest())
        sigs.append(goasn1.marshal_ecdsa_signature(int.from_bytes(bytes(r), "big"), int.from_bytes(bytes(s), "big")))
    sig_ok = np.zeros(max(J, 1), np.uint8)
    if live:
        soff = np.zeros(len(live) + 1, np.uint32); soff[1:] = np.cumsum([len(x) for x in sigs])
        st = fast.verify_batch(keys, np.array(key_idx, np.int32), np.frombuffer(b"".join(digs), np.uint8), (np.arange(len(live) + 1) * 32).astype(np.uint32),
                               np.frombuffer(b"".join(sigs), np.uint8), soff, nthreads=4)
        sig_ok[np.array(live)] = (st == o.VALID)
    chk = np.zeros((max(T, 1), 2, 32), np.uint8)
    for t in range(T):
        L.bd_check(h, t, segs)
        chk[t, 0] = np.frombuffer(hashlib.sha256(msg(segs, 0)).digest(), np.uint8)
        chk[t, 1] = np.frombuffer(hashlib.sha256(msg(segs, 6)).digest(), np.uint8)
    pbits = np.zeros((0, len(principals)), bool) if principal_bits is None else np.asarray(principal_bits, bool)
    words = np.ascontiguousarray(pkg().binding.pack_principal_bits(pbits), np.uint32).reshape(-1)
    flags = np.full(max(T, 1), 254, np.uint8)
    ckeys = sorted(collections) if collections else []
    cnb, cno = _blob([ns.encode() for ns, _ in ckeys])
    ccb, cco = _blob([c.encode() for _, c in ckeys])
    croots = np.array([collections[k] for k in ckeys] or [0], np.int32)
    rc = L.txid_decide(kt.h, h, ts.h if ts is not None else None, mode, _p(vb), _p(vo) if versions is not None else None, _p(sig_ok), _p(chk),
                       _p(words if words.size else np.zeros(1, np.uint32)), pbits.shape[0], pbits.shape[1],
                       _p(cnb), _p(cno), _p(ccb), _p(cco), _p(croots), len(ckeys), _p(flags))
    L.bd_free(h)
    if rc:
        raise ValueError("a (namespace, collection) pair is given twice")
    return flags[:T]
