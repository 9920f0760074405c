"""The device-side block logic run on the host with a channel capability: klutil.device_logic_flags over the host build of
tests/host_sim/blockdev_v13_host.cpp, whose walk and decide stage take the mode fabgpu_channel_capability selects and the versions
fabgpu_namespace_versions installs, and which applies the block's lscc pass after the duplicate pass."""
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
import klutil

MODE_V20, MODE_V13 = 0, 1
_LIB = None


def v13_lib():
    """built into a temporary directory: the source tree is not written"""
    global _LIB
    if _LIB is None:
        d = os.path.join(ROOT, "tests", "host_sim")
        so = os.path.join(tempfile.mkdtemp(prefix="fabgpu_v13_"), "libblockdev_v13_host.so")
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-o", so, os.path.join(d, "blockdev_v13_host.cpp"),
                               os.path.join(ROOT, "fabric-mod_b200", "csrc", "blockval.cpp")])
        _LIB = ctypes.CDLL(so)
        _LIB.bd_new.restype = ctypes.c_void_p
        _LIB.kl_new.restype = ctypes.c_void_p
        _LIB.kl_apply.restype = ctypes.c_char_p
    return _LIB


class _KeyTable(klutil.KeyTable):
    def __init__(self, base_nodes, n_principals):
        self.L = v13_lib()
        self.h = ctypes.c_void_p(self.L.kl_new())
        self.base, self.np = base_nodes, n_principals


def device_flags(env_blob, env_off, identities, channel, nodes, principals, mode=MODE_V13, policies=None, versions=None, principal_bits=None,
                 collections=None, key_calls=(), writes_hint=32, out=None):
    """Flags of the host build.  policies: {namespace: root} (installed sorted by name, as the binding does); versions: {namespace:
    version} for those entries (missing: no version; None: none installed).  out (dict) receives 'lscc_seen'."""
    from oracle import goasn1
    L = v13_lib()
    nodes = np.ascontiguousarray(nodes, np.int32).reshape(-1, 4)
    kt = _KeyTable(nodes.shape[0], len(principals))
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
    conf = np.zeros(max(T, 1), np.uint8)
    ckeys = sorted(collections) if collections else []
    cnb, cno = _blob([ns.encode() for ns, _ in ckeys])
    ccb, cco = _blob([c.encode() for _, c in ckeys])
    croots = np.array([collections[k] for k in ckeys] or [0], np.int32)
    seen = ctypes.c_int(0)
    rc = L.v13_decide(kt.h, h, mode, _p(vb), _p(vo) if versions is not None else None, _p(sig_ok), _p(chk),
                      _p(words if words.size else np.zeros(1, np.uint32)), pbits.shape[0], pbits.shape[1],
                      _p(cnb), _p(cno), _p(ccb), _p(cco), _p(croots), len(ckeys), _p(flags), _p(conf), ctypes.byref(seen))
    L.bd_free(h)
    if rc:
        raise ValueError("a (namespace, collection) pair is given twice")
    if out is not None:
        out["lscc_seen"] = bool(seen.value)
    return flags[:T]
