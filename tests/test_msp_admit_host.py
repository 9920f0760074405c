"""Identity admission's host logic and the unknown-identity listing on the host build (tests/host_sim/msp_admit_host.cpp): the MSP
table's mirror under random configure / add / grow sequences, and the listing steps of unknownids.cuh against identity_oracle on
seeded blocks, on two identities with one sample_hash, and on the wire-mutation corpus -- plus the same listing under AddressSanitizer
and UndefinedBehaviorSanitizer."""
import ctypes
import os
import random
import struct
import subprocess
import tempfile

import numpy as np
import pytest

from tools import blockgen
from tools import fabricpb as pb
from util import ROOT
from blockutil import _blob
import identity_oracle as io
import wiremut

SRC = os.path.join(ROOT, "tests", "host_sim", "msp_admit_host.cpp")
_LIB = None


def _p(a):
    return a.ctypes.data_as(ctypes.c_void_p) if a is not None else None


def lib():
    """built into a temporary directory: the source tree is not written"""
    global _LIB
    if _LIB is None:
        so = os.path.join(tempfile.mkdtemp(prefix="fabgpu_admit_"), "libmsp_admit_host.so")
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-o", so, SRC])
        L = ctypes.CDLL(so)
        L.mm_new.restype = ctypes.c_void_p
        L.mm_free.argtypes = [ctypes.c_void_p]
        L.mm_configure.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int]
        L.mm_add.restype = ctypes.c_char_p
        L.mm_add.argtypes = [ctypes.c_void_p] + [ctypes.c_void_p] * 8 + [ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.POINTER(ctypes.c_int)]
        L.mm_find.argtypes = [ctypes.c_void_p, ctypes.c_char_p, ctypes.c_uint32]
        L.mm_info.argtypes = [ctypes.c_void_p, ctypes.c_void_p]
        L.uk_list.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_uint32, ctypes.c_char_p, ctypes.c_void_p, ctypes.c_uint32,
                              ctypes.POINTER(ctypes.c_uint32)]
        _LIB = L
    return _LIB


class Mirror:
    def __init__(self, ids):
        self.L = lib()
        self.h = ctypes.c_void_p(self.L.mm_new())
        b, o = _blob(ids)
        self.L.mm_configure(self.h, _p(b), _p(o), len(ids))

    def add(self, ids, group=None, bits=None, groups_on=False, bits_on=False, n=None, off=None):
        """None on success, else the refusal text"""
        b, o = _blob(ids)
        if off is not None:
            o = np.asarray(off, np.uint32)
        mb, mo = _blob([b"Org1MSP"] * len(ids))
        keys = np.zeros(64 * max(len(ids), 1), np.uint8)
        valid = np.ones(max(len(ids), 1), np.uint8)
        g = None if group is None else np.asarray(list(group) or [0], np.int32)
        w = None if bits is None else np.asarray(list(bits) or [0], np.uint32)
        grew = ctypes.c_int(0)
        err = self.L.mm_add(self.h, _p(b), _p(o), _p(mb), _p(mo), _p(keys), _p(valid), _p(g), _p(w), len(ids) if n is None else n,
                            int(groups_on), int(bits_on), ctypes.byref(grew))
        return err.decode() if err else None

    def find(self, ser):
        return self.L.mm_find(self.h, ser, len(ser))

    def info(self):
        out = np.zeros(3, np.uint64)
        self.L.mm_info(self.h, _p(out))
        return [int(x) for x in out]

    def listing(self, block, env_off, channel):
        env_off = np.ascontiguousarray(env_off, np.uint32)
        n_env = env_off.shape[0] - 1
        buf = np.frombuffer(bytes(block) + bytes(64), np.uint8)
        cap = 17 * max(n_env, 1)
        out = np.zeros(3 * cap, np.uint32)
        n = ctypes.c_uint32(0)
        self.L.uk_list(self.h, _p(buf), _p(env_off), n_env, channel.encode(), _p(out), cap, ctypes.byref(n))
        return [(int(out[3 * i]), int(out[3 * i + 1]), int(out[3 * i + 2])) for i in range(n.value)]

    def __del__(self):
        self.L.mm_free(self.h)


def _ident(r, k):
    """a serialized identity of the size and shape of a client certificate"""
    return pb.serialized_identity("Org%dMSP" % (1 + k % 4), blockgen._pem_blob(b"id%d-%d" % (k, r.randrange(1 << 30))))


def test_mirror_random_sequences():
    """Random configure / add / grow sequences: after every step the mirror finds every identity it holds and nothing else, its
    load stays below 1/4, growth doubles, and every refusal leaves it unchanged."""
    r = random.Random(11)
    for seq in range(6):
        held = [_ident(r, k) for k in range(r.choice([0, 1, 5, 40]))]
        m = Mirror(held)
        outside = [_ident(r, 10 ** 6 + k) for k in range(20)]
        for step in range(40):
            kind = r.random()
            if kind < 0.15:                                           # a refusal: the mirror must not change
                before = m.info()
                dup = r.choice(held) if held else _ident(r, 5)
                fresh = _ident(r, 2 * 10 ** 6 + step)
                cases = [([fresh, fresh], {}), ([fresh, b""], {}), ([fresh], dict(group=[0])), ([fresh], dict(bits=[0])),
                         ([fresh], dict(groups_on=True)), ([fresh], dict(bits_on=True)), ([fresh], dict(group=[-1], groups_on=True)),
                         ([fresh, fresh + b"x"], dict(off=[0, len(fresh), 3])), ([fresh], dict(n=-1))]
                if held:
                    cases.append(([fresh, dup], {}))
                ids, kw = r.choice(cases)
                assert m.add(ids, **kw) is not None
                assert m.info() == before
                assert m.find(fresh) == -1
                continue
            new = [_ident(r, 3 * 10 ** 6 + 100 * step + k) for k in range(r.choice([1, 2, 7, 30, 200]))]
            size0 = m.info()[1]
            assert m.add(new) is None
            held += new
            n, size, occupied = m.info()
            assert n == len(held) == occupied
            assert 4 * n + 8 <= size and size & (size - 1) == 0
            assert size == size0 or size >= 2 * size0
            for i, ser in enumerate(held):
                assert m.find(ser) == i
            for ser in outside:
                assert m.find(ser) == -1


def _net_block(n_tx, seed, unknown_every=3, n_clients=12):
    """A block of n_tx well-formed transactions whose creators and endorsers include identities the table does not hold"""
    net = blockgen.Network(n_orgs=4, n_clients=n_clients, seed=seed)
    faults = {t: "unknown_endorser" for t in range(1, n_tx, unknown_every)}
    faults.update({t: "unknown_creator" for t in range(2, n_tx, 2 * unknown_every)})
    faults.update({t: "same_cert_two_encodings" for t in range(0, n_tx, 5)})
    blk, info = blockgen.build_block(net, n_tx, 3, faults, seed=seed, nthreads=2)
    return net, blk, info


@pytest.mark.parametrize("seed", [1, 2, 3])
def test_listing_matches_the_oracle_on_seeded_blocks(seed):
    """Half the clients and half the alternative peer encodings configured: the host build lists what identity_oracle lists, with
    offsets into the envelope blob that hold exactly those bytes."""
    net, blk, info = _net_block(60, seed)
    held = [i.serialized for i in net.peers + net.clients[::2] + [net.invalid_cert] + net.peers_alt[:2]]
    m = Mirror(held)
    envs = io.envelopes(info)
    got = m.listing(info["env_blob"], info["env_off"], net.channel)
    exp = io.listing(envs, held)
    assert len(exp) > 5
    assert [(bytes(info["env_blob"][o:o + ln]), t) for o, ln, t in got] == exp
    # the same block after admitting what was listed: nothing left
    assert m.add([s for s, _ in exp]) is None
    assert m.listing(info["env_blob"], info["env_off"], net.channel) == []


def _collide(ser: bytes) -> bytes:
    """another identity with the same sample_hash: one byte changed outside the sampled windows (head 16, the 32 around the middle,
    [n - 72, n - 40), tail 24)"""
    n = len(ser)
    assert n >= 160
    i = 20
    assert i < n // 2 - 16
    b = bytearray(ser)
    b[i] ^= 0x01
    return bytes(b)


def test_listing_keeps_identities_with_one_hash_apart():
    """Two distinct unknown creators with equal sample_hash both appear, each once, in first-appearance order."""
    net = blockgen.Network(n_orgs=4, n_clients=2, seed=9)
    twin = blockgen.Identity(net.clients[1].mspid, net.clients[1].priv_index, net.clients[1].xy, net.clients[1].cert_pem)
    twin.serialized = _collide(net.clients[1].serialized)
    assert twin.serialized != net.clients[1].serialized
    net.clients = [net.clients[0], net.clients[1], twin, net.clients[1], twin]
    blk, info = blockgen.build_block(net, 10, 3, {}, seed=4, nthreads=2)
    held = [i.serialized for i in net.peers + [net.clients[0]]]
    m = Mirror(held)
    got = [(bytes(info["env_blob"][o:o + ln]), t) for o, ln, t in m.listing(info["env_blob"], info["env_off"], net.channel)]
    assert got == io.listing(io.envelopes(info), held) == [(net.clients[1].serialized, 1), (twin.serialized, 2)]


def _check_ranges(got, envs, blob, held):
    """Every listed range lies inside the blob, names a creator or endorser field the oracle parse of that transaction sees (when it
    parses), is not held, and is listed once, in non-decreasing first-tx order.  An endorsement without an endorser is a lookup of
    the empty identity, and is listed as such."""
    seen = set()
    last = 0
    for off, ln, t in got:
        assert off + ln <= len(blob)
        ser = bytes(blob[off:off + ln])
        assert ser not in held and ser not in seen
        seen.add(ser)
        assert t >= last
        last = t
        looked = io.lookups(envs[t])
        if looked is not None:
            assert ser in looked


def test_listing_on_the_wire_mutation_corpus():
    """The corpus with only the peers configured: every listing is well formed, and on the transactions the oracle parses fully it is
    the oracle's."""
    net, ids, nodes, pol, blocks = wiremut.corpus()
    held = {i.serialized for i in net.peers}
    m = Mirror(sorted(held))
    total = 0
    for blk, info, labels, _ in blocks:
        envs = io.envelopes(info)
        got = m.listing(info["env_blob"], info["env_off"], net.channel)
        _check_ranges(got, envs, info["env_blob"], held)
        total += len(got)
        clean = [e for e in envs if io.lookups(e) is not None]
        assert clean
    assert total > 0


def _corpus_file(path, records):
    u32 = lambda v: struct.pack("<I", v)
    out = u32(len(records))
    for held, channel, blob, env_off in records:
        out += u32(len(held)) + b"".join(u32(len(h)) + h for h in held)
        out += u32(len(channel)) + channel.encode() + u32(len(blob)) + bytes(blob) + u32(len(env_off) - 1) + b"".join(u32(int(x)) for x in env_off)
    path.write_bytes(out)


def test_listing_under_sanitizers(tmp_path):
    exe = str(tmp_path / "uk_asan")
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-g", "-fsanitize=address,undefined", "-fno-sanitize-recover=all", "-fno-omit-frame-pointer",
                           "-DUK_ASAN_MAIN", "-o", exe, SRC])
    net, ids, nodes, pol, blocks = wiremut.corpus()
    held = sorted({i.serialized for i in net.peers})
    records = [(held, net.channel, info["env_blob"], info["env_off"]) for _, info, _, _ in blocks]
    snet, sblk, sinfo = _net_block(40, 5)
    sheld = [i.serialized for i in snet.peers + snet.clients[::2]]
    records.append((sheld, snet.channel, sinfo["env_blob"], sinfo["env_off"]))
    path = tmp_path / "corpus.bin"
    _corpus_file(path, records)
    env = dict(os.environ, ASAN_OPTIONS="detect_leaks=0:halt_on_error=1", UBSAN_OPTIONS="halt_on_error=1:print_stacktrace=1")
    res = subprocess.run([exe, str(path)], capture_output=True, text=True, env=env)
    assert res.returncode == 0, res.stderr[-4000:]
    lines = res.stdout.splitlines()
    assert len(lines) == len(records)
    for line, (h, ch, blob, off) in zip(lines, records):
        v = [int(x) for x in line.split()]
        got = [tuple(v[i:i + 3]) for i in range(0, len(v), 3)]
        assert got == Mirror(h).listing(blob, off, ch)
        _check_ranges(got, [bytes(blob[off[t]:off[t + 1]]) for t in range(len(off) - 1)], blob, set(h))
    last = [int(x) for x in lines[-1].split()]
    assert [(bytes(sinfo["env_blob"][last[i]:last[i] + last[i + 1]]), last[i + 2]) for i in range(0, len(last), 3)] == \
        io.listing(io.envelopes(sinfo), sheld)
