"""Shared helpers for the block-validation tests."""
import ctypes
import hashlib
import os
import subprocess

import numpy as np

from oracle import bccsp_sw as o
from oracle import fast
from tools import blockgen
from util import ROOT


def identities_of(net):
    return [(i.serialized, i.mspid, i.xy, i.valid) for i in net.msp_table]


def fault_map(n_tx, stride=3, start=2):
    """Every fault once, separated by valid transactions (dup_txid needs a valid predecessor)."""
    faults = {}
    t = start
    for f in blockgen.FAULTS:
        if t >= n_tx:
            break
        faults[t] = f
        t += stride
    return faults


def _blob(items):
    off = np.zeros(len(items) + 1, np.uint32)
    off[1:] = np.cumsum([len(x) for x in items])
    return np.ascontiguousarray(np.frombuffer(b"".join(items) or b"\x00", np.uint8)), off


def _p(a):
    return a.ctypes.data_as(ctypes.c_void_p)


_BD = None


def bd_lib():
    global _BD
    if _BD is None:
        d = os.path.join(ROOT, "tests", "host_sim")
        so, src = os.path.join(d, "libblockdev_host.so"), os.path.join(d, "blockdev_host.cpp")
        csrc = os.path.join(ROOT, "fabric-mod_b200", "csrc")
        deps = [src] + [os.path.join(csrc, f) for f in ("blockdev.cuh", "blockval.cpp", "blockval.hpp")]
        if not os.path.exists(so) or any(os.path.getmtime(so) < os.path.getmtime(f) for f in deps):
            subprocess.check_call(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-o", so, src, os.path.join(csrc, "blockval.cpp")])
        _BD = ctypes.CDLL(so)
        _BD.bd_new.restype = ctypes.c_void_p
        _BD.bd_split_block.argtypes = [ctypes.c_void_p, ctypes.c_size_t, ctypes.c_void_p, ctypes.c_int]
    return _BD


def split_block(blk: bytes):
    """The library's split_block (blockval.cpp) on a serialized Block: the envelopes, or None when the Block does not parse."""
    L = bd_lib()
    buf = np.frombuffer(blk or b"\x00", np.uint8)
    cap = len(blk) + 1
    out = np.zeros(2 * cap, np.uint32)
    n = L.bd_split_block(_p(buf), len(blk), _p(out), cap)
    return None if n < 0 else [blk[out[2 * i]: out[2 * i] + out[2 * i + 1]] for i in range(n)]


def device_logic_flags(env_blob, env_off, identities, channel, nodes, principals, policies=None):
    """The device-side block logic (blockdev.cuh) executed on the host, driven by oracle verdicts and hashlib digests.
    policies: {namespace: root node} (None: one policy for every namespace)."""
    return device_logic_run(env_blob, env_off, identities, channel, nodes, principals, policies)[0]


def device_logic_run(env_blob, env_off, identities, channel, nodes, principals, policies=None, ends_hint=16, poison=False):
    """device_logic_flags with the job arrays sized T (1 + ends_hint) and, with poison, filled with garbage instead of dead records
    before the walk.  -> (flags, number of job slots the later stages would read that the walk left unwritten)."""
    from oracle import goasn1
    from util import pkg
    L = bd_lib()
    idb, ido = _blob([bytes(i[0]) for i in identities])
    mb, mo = _blob([i[1].encode() for i in identities])
    keys = np.ascontiguousarray(np.frombuffer(b"".join(bytes(i[2]) for i in identities), np.uint8)).reshape(-1, 64)
    valid = np.array([1 if i[3] else 0 for i in identities], np.uint8)
    nodes = np.ascontiguousarray(nodes, np.int32)
    pbb, pbo = _blob([p.encode() for p in principals])
    h = ctypes.c_void_p(L.bd_new(_p(idb), _p(ido), _p(mb), _p(mo), _p(valid), len(identities), _p(nodes), nodes.shape[0], _p(pbb), _p(pbo),
                                 len(principals), channel.encode()))
    groups = np.ascontiguousarray(pkg().binding.identity_groups(identities), np.int32)      # product code: Mspid + certificate groups
    L.bd_groups(h, _p(groups), len(identities))
    if policies:
        names = sorted(policies)
        nb, no = _blob([n.encode() for n in names])
        roots = np.array([policies[n] for n in names], np.int32)
        L.bd_namespaces(h, _p(nb), _p(no), _p(roots), len(names))
    blob = np.frombuffer(env_blob, np.uint8) if len(env_blob) else np.zeros(1, np.uint8)
    env_off = np.ascontiguousarray(env_off, np.uint32)
    T = env_off.shape[0] - 1
    n_end = L.bd_plan_ex(h, _p(blob), _p(env_off), T, ends_hint, 1 if poison else 0)
    stale = L.bd_stale(h)
    J = T + n_end
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
    flags = np.full(max(T, 1), 254, np.uint8)
    L.bd_decide(h, _p(sig_ok), _p(chk), _p(flags))
    L.bd_free(h)
    return flags[:T], stale


def device_gate(sig: bytes):
    """-> (ok, r32, s32, status) from the device-side gate functions run on the host."""
    L = bd_lib()
    r = (ctypes.c_uint8 * 32)(); s = (ctypes.c_uint8 * 32)()
    buf = (ctypes.c_uint8 * max(1, len(sig))).from_buffer_copy(sig if sig else b"\x00")
    ok = L.bd_gate(buf, ctypes.c_uint32(len(sig)), r, s)
    st = L.bd_gate_status(buf, ctypes.c_uint32(len(sig)), r, s)
    return bool(ok), bytes(r), bytes(s), int(st)


def capacity_edge_cases():
    """Capacity edges of the device logic: BD_MAX_NS_SEEN (8 / 9 namespaces), BD_MAX_NS (4 / 5 written namespaces), BD_MAX_SIGNERS
    (64 / 65 distinct verified signers).  [(name, network, n_tx, nodes, policies, build_block shape, index of the transaction at the
    limit, index of the one past it)]."""
    cc = blockgen.CHAINCODE
    net = blockgen.Network()
    nodes = net.policy_n_of(2)
    seen = lambda t: [(cc, 1, 1)] + [("read%d" % i, 1, 0) for i in range(7 + (t == 1))]            # 8 / 9 namespaces
    wrote = lambda t: [(cc, 1, 1)] + [("write%d" % i, 0, 1) for i in range(3 + (t == 1))]          # 4 / 5 written namespaces
    pol = {cc: 0, **{"write%d" % i: 0 for i in range(4)}}
    many = blockgen.Network(n_orgs=4, n_clients=70, seed=0x5167)
    signers = lambda t: many.clients[: 64 + (t == 1)] if t < 2 else [many.peers[(t + k) % 4] for k in range(3)]   # 64 / 65 signers
    return [("namespaces_seen", net, 4, nodes, {cc: 0}, dict(namespaces=seen), 0, 1),
            ("namespaces_written", net, 4, nodes, pol, dict(namespaces=wrote), 0, 1),
            ("signers", many, 12, many.policy_n_of(3), None, dict(endorsers=signers), 0, 1)]
