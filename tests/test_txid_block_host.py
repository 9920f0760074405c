"""fabgpu_committed_txids_add_block's device logic in the tests' host build (tests/host_sim/txid_block_host.cpp): the id extractor and the
block insert that txid_block_id_kernel / txid_block_insert_kernel run, against txid_block_oracle on the cases, the wire-mutation corpus
and seeded random blocks; and the set add_block leaves against the set _add of the oracle's ids leaves."""
import ctypes
import os
import subprocess
import tempfile

import numpy as np
import pytest

from tools import blockgen
from util import ROOT
from blockutil import _p
import txid_block_oracle as tbo
import txidblockcases
import txidutil
import wiremut

_LIB = None


def lib():
    """txidutil's host library plus the add_block code, built into a temporary directory; txidutil.HostSet runs on it"""
    global _LIB
    if _LIB is None:
        d = os.path.join(ROOT, "tests", "host_sim")
        so = os.path.join(tempfile.mkdtemp(prefix="fabgpu_txidblock_"), "libtxid_block_host.so")
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-o", so, os.path.join(d, "txid_block_host.cpp"),
                               os.path.join(ROOT, "fabric-mod_b200", "csrc", "blockval.cpp")])
        L = ctypes.CDLL(so)
        L.txs_new.restype = ctypes.c_void_p
        L.txs_new.argtypes = [ctypes.c_ulonglong]
        L.txs_apply.restype = ctypes.c_char_p
        L.txs_apply.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_size_t, ctypes.c_size_t,
                                ctypes.c_ulonglong, ctypes.POINTER(ctypes.c_int)]
        L.txs_info.argtypes = [ctypes.c_void_p, ctypes.c_void_p]
        L.txs_lookup.argtypes = [ctypes.c_void_p, ctypes.c_char_p]
        L.txs_free.argtypes = [ctypes.c_void_p]
        L.txb_extract.argtypes = [ctypes.c_void_p, ctypes.c_size_t, ctypes.c_void_p, ctypes.c_uint32, ctypes.c_void_p, ctypes.c_void_p]
        L.txs_add_block.restype = ctypes.c_char_p
        L.txs_add_block.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_size_t, ctypes.c_void_p, ctypes.c_uint32, ctypes.c_ulonglong,
                                    ctypes.POINTER(ctypes.c_int), ctypes.POINTER(ctypes.c_uint)]
        _LIB = L
    return _LIB


class Set(txidutil.HostSet):
    def __init__(self, seed=0x5EED, max_bytes=0):
        self.L = lib()
        self.h = ctypes.c_void_p(self.L.txs_new(seed))
        self.max_bytes = max_bytes

    def add_block(self, envs):
        blob, off = _assemble(envs)
        failed, inserting = ctypes.c_int(0), ctypes.c_uint(0)
        err = self.L.txs_add_block(self.h, _p(blob), blob.shape[0], _p(off), len(envs), self.max_bytes, ctypes.byref(failed), ctypes.byref(inserting))
        if err is not None:
            raise txidutil.SetError(err.decode(), bool(failed.value))
        return inserting.value


def _assemble(envs):
    off = np.zeros(len(envs) + 1, np.uint32)
    off[1:] = np.cumsum([len(e) for e in envs])
    blob = np.frombuffer(b"".join(envs) or b"\0", np.uint8).copy()
    return blob, off


def extract(envs):
    """per envelope: the canonical id the device extracts (str), or None"""
    blob, off = _assemble(envs)
    T = len(envs)
    kind = np.zeros(max(T, 1), np.uint8)
    ids = np.zeros((max(T, 1), 32), np.uint8)
    lib().txb_extract(_p(blob), blob.shape[0], _p(off), T, _p(kind), _p(ids))
    return [bytes(ids[t]).hex() if kind[t] else None for t in range(T)]


def _oracle_ids(envs):
    out = []
    for e in envs:
        i = tbo.block_store_id(e)
        out.append(i.decode() if tbo.canonical(i) else None)
    return out


def _state(s, id_str):
    return s.lookup(bytes.fromhex(id_str))


def test_cases_extract_the_ids_written_out():
    cases = txidblockcases.cases()
    envs = [e for _, e, _ in cases]
    got = extract(envs)
    for (name, e, exp), g in zip(cases, got):
        assert g == exp, name
        assert _oracle_ids([e])[0] == exp, name


def _check_block(envs, installed=None):
    """add_block on a set holding `installed` ({id: kind}) == _add of the oracle's ids on another"""
    installed = dict(installed or {"0" * 64: 0})
    a, b = Set(), Set()
    for s in (a, b):
        s.apply(True, list(installed), list(installed.values()))
    n = a.add_block(envs)
    ids = tbo.indexed_ids(envs)
    b.apply(False, ids)
    assert n == len(ids)
    assert a.info()[0] == b.info()[0] == len(tbo.after(installed, [envs]))
    table = tbo.after(installed, [envs])
    for i, k in table.items():
        assert _state(a, i) == _state(b, i) == 2 + k, i
    return a


def test_cases_add_block_and_kind_1_stays():
    envs = [e for _, e, _ in txidblockcases.cases()]
    _check_block(envs)
    _check_block(envs, {txidblockcases.PLAIN: 1, txidblockcases.COMPUTED: 1, "0" * 64: 0})


def test_in_block_duplicates_insert_once():
    envs = [c[1] for c in txidblockcases.cases()]
    s = _check_block(envs * 3 + envs[::-1])
    assert s.info()[0] == 1 + len(tbo.indexed_ids(envs))


def test_wire_mutation_corpus():
    net, ids, nodes, pol, blocks = wiremut.corpus()
    for blk, info, labels, _ in blocks:
        off = info["env_off"]
        envs = [bytes(info["env_blob"][off[t]:off[t + 1]]) for t in range(off.shape[0] - 1)]
        got, exp = extract(envs), _oracle_ids(envs)
        for t in range(len(envs)):
            assert got[t] == exp[t], (t, labels[t])
        _check_block(envs)


@pytest.mark.parametrize("seed", [3, 4, 5])
def test_seeded_random_blocks(seed):
    """blockgen blocks with faults, emptied tx ids, random bytes and replays, as a sequence of blocks on one set"""
    rng = np.random.default_rng(seed)
    net = blockgen.Network()
    n = 120
    s, table = Set(), {"0" * 64: 0}
    s.apply(True, list(table))
    prev = []
    for k in range(4):
        blk, info = blockgen.build_block(net, n, 2, None, seed=seed * 10 + k, number=k + 1, nthreads=2)
        off = info["env_off"]
        envs = [bytes(info["env_blob"][off[t]:off[t + 1]]) for t in range(n)]
        for t in rng.choice(n, 10, replace=False):
            envs[t] = txidblockcases.with_txid(envs[t], "")
        for t in rng.choice(n, 5, replace=False):
            b = bytearray(envs[t]); b[rng.integers(0, len(b))] ^= 1 << int(rng.integers(0, 8)); envs[t] = bytes(b)
        envs += [bytes(rng.integers(0, 256, int(rng.integers(0, 40)), dtype=np.uint8)) for _ in range(5)]
        envs += prev[:10]
        rng.shuffle(envs)
        assert extract(envs) == _oracle_ids(envs)
        s.add_block(envs)
        table = tbo.after(table, [envs])
        assert s.info()[0] == len(table)
        for i in table:
            assert _state(s, i) == 2
        prev = envs


def test_refusals_and_growth():
    s = Set()
    with pytest.raises(txidutil.SetError, match="no committed tx-id set"):
        s.add_block([txidblockcases.cases()[0][1]])
    s.apply(True, ["0" * 64])
    assert s.info() == (1, 1024)
    net = blockgen.Network()
    for k in range(3):
        _, info = blockgen.build_block(net, 700, 2, None, seed=90 + k, number=k + 1, nthreads=2)
        off = info["env_off"]
        s.add_block([bytes(info["env_blob"][off[t]:off[t + 1]]) for t in range(700)])
    assert s.info() == (2101, 8192)
    b = Set(max_bytes=36 * 1024)
    b.apply(True, ["0" * 64])
    with pytest.raises(txidutil.SetError) as e:
        b.add_block([bytes(info["env_blob"][off[t]:off[t + 1]]) for t in range(700)])
    assert e.value.failed
    with pytest.raises(txidutil.SetError, match="broken"):
        b.add_block([txidblockcases.cases()[0][1]])
