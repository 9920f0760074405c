"""The committed tx-id set (fabgpu_committed_txids) in the device block logic, run on the host build
(tests/host_sim/blockdev_txid_host.cpp): the cases' written-out codes, the oracle on the fault corpus, and the table's own logic --
canonical filter, argument checks, de-duplication, kinds, growth, and probe chains of ids that share a long prefix."""
import hashlib

import numpy as np
import pytest

from oracle import blockval as ob
from tools import blockgen
import blockutil
import collcases
import klcases
import txid_oracle
import txidcases
import txidutil


def _run(case, use_bits):
    net, blk, info, codes, calls, table = txidcases.materialize(case)
    names, bits = collcases.principals(use_bits)
    kt = klcases.key_table((case[0], False, {}, case[3])) if case[2] else None
    ids = net.identities()
    host = txidutil.device_flags(info["env_blob"], info["env_off"], ids, net.channel, collcases.forest()[0], names, mode=case[1],
                                 policies=txidcases.policies(), versions=txidcases.versions(), principal_bits=bits,
                                 key_calls=[(True,) + kt] if kt else (), txid_calls=calls)
    exp = txidcases.oracle_flags(case, blk, net, names, bits, table)
    return host.tolist(), exp.tolist(), codes


@pytest.mark.parametrize("use_bits", [True, False], ids=["bits", "msp_ids"])
@pytest.mark.parametrize("case", txidcases.cases(), ids=lambda c: c[0])
def test_txid_case_host_build(case, use_bits):
    """Every case: the oracle and the host build give the codes written out."""
    host, exp, codes = _run(case, use_bits)
    assert exp == codes
    assert host == codes


@pytest.mark.parametrize("case", txidcases.cases(), ids=lambda c: c[0])
def test_no_set_is_the_parent_behaviour(case):
    """Without a set installed, the host build and the oracle give what they give without the ledger check."""
    net, blk, info, codes, calls, table = txidcases.materialize(case)
    names, bits = collcases.principals(True)
    kt = klcases.key_table((case[0], False, {}, case[3])) if case[2] else None
    host = txidutil.device_flags(info["env_blob"], info["env_off"], net.identities(), net.channel, collcases.forest()[0], names, mode=case[1],
                                 policies=txidcases.policies(), versions=txidcases.versions(), principal_bits=bits,
                                 key_calls=[(True,) + kt] if kt else (), txid_calls=None)
    exp = txidcases.oracle_flags(case, blk, net, names, bits, None)
    assert host.tolist() == exp.tolist()
    empty = txidutil.device_flags(info["env_blob"], info["env_off"], net.identities(), net.channel, collcases.forest()[0], names, mode=case[1],
                                  policies=txidcases.policies(), versions=txidcases.versions(), principal_bits=bits,
                                  key_calls=[(True,) + kt] if kt else (), txid_calls=[(True, [], None), (True, ["x"], None)])
    assert empty.tolist() == host.tolist()


def test_fault_corpus_with_half_the_ids_committed():
    """The blockgen fault corpus with a set holding about half of the block's ids (a third of those as kind 1): host build == oracle, in
    both modes."""
    import nodeou
    net = nodeou.network(4)
    n = 3 * len(blockgen.FAULTS) + 4
    faults = blockutil.fault_map(n)
    blk, info = blockgen.build_block(net, n, 3, faults, seed=5, nthreads=2, endorsers=lambda t: [net.org_peers[o][0] for o in (t % 4, (t + 1) % 4)])
    envs = [bytes(info["env_blob"][info["env_off"][t]:info["env_off"][t + 1]]) for t in range(n)]
    ids = [txid_oracle.txid_of(e) for e in envs]
    rng = np.random.default_rng(3)
    chosen = [t for t in range(n) if ids[t] is not None and rng.random() < 0.5]
    kinds = [1 if k % 3 == 0 else 0 for k in range(len(chosen))]
    table = {}
    for t, k in zip(chosen, kinds):
        table[ids[t]] = max(table.get(ids[t], 0), k)
    names, bits = collcases.principals(True)
    moved = 0
    for mode in (txidcases.MODE_V20, txidcases.MODE_V13):
        case = ("corpus", mode, False, [])
        host = txidutil.device_flags(info["env_blob"], info["env_off"], net.identities(), net.channel, collcases.forest()[0], names, mode=mode,
                                     policies=txidcases.policies(), versions=txidcases.versions(), principal_bits=bits,
                                     txid_calls=[(True, [ids[t] for t in chosen], kinds)])
        exp = txidcases.oracle_flags(case, blk, net, names, bits, table)
        base = txidcases.oracle_flags(case, blk, net, names, bits, None)
        assert host.tolist() == exp.tolist()
        moved += int((exp != base).sum())
    assert moved >= 10


# ---- the table on its own -------------------------------------------------------------------------------------------------------
def _hex(b):
    return bytes(b).hex()


def test_canonical_filter():
    L = txidutil.txid_lib()
    out = (np.zeros(32, np.uint8))
    good = hashlib.sha256(b"x").hexdigest()
    assert L.txs_canonical(good.encode(), 64, out.ctypes.data) == 1 and bytes(out) == hashlib.sha256(b"x").digest()
    for bad in (good.upper(), good[:63], good + "0", "", "g" * 64, good[:62] + " a", good[:63] + "\x00"):
        assert L.txs_canonical(bad.encode(), len(bad.encode()), out.ctypes.data) == 0, bad
    s = txidutil.HostSet()
    s.apply(True, [good.upper(), good[:63], good + "0", "", "G" * 64])
    assert s.info()[0] == 0
    assert s.lookup(hashlib.sha256(b"x").digest()) == 0


def test_argument_refusals_keep_the_set():
    s = txidutil.HostSet()
    with pytest.raises(txidutil.SetError, match="no committed tx-id set installed"):
        s.apply(False, [hashlib.sha256(b"a").hexdigest()])
    ids = [hashlib.sha256(b"%d" % k).hexdigest() for k in range(10)]
    s.apply(True, ids)
    with pytest.raises(txidutil.SetError, match="kind") as e:
        s.apply(False, ids[:2], [0, 2])
    assert not e.value.failed
    L = txidutil.txid_lib()
    import ctypes
    failed = ctypes.c_int(0)
    blob = np.frombuffer(("".join(ids[:2])).encode(), np.uint8)
    dec = np.array([0, 64, 10], np.uint32)
    assert b"decrease" in L.txs_apply(s.h, 0, blob.ctypes.data, dec.ctypes.data, None, 2, 0, 0, ctypes.byref(failed))
    assert b"missing" in L.txs_apply(s.h, 0, None, None, None, 2, 0, 0, ctypes.byref(failed))
    assert s.info()[0] == 10
    for k in range(10):
        assert s.lookup(hashlib.sha256(b"%d" % k).digest()) == 2


def test_kinds_duplicates_within_a_call_and_the_larger_kind():
    s = txidutil.HostSet()
    a, b, c = (hashlib.sha256(x).hexdigest() for x in (b"a", b"b", b"c"))
    s.apply(True, [a, a, b, b, c], [0, 1, 1, 0, 0])
    assert s.info()[0] == 3
    assert [s.lookup(bytes.fromhex(x)) for x in (a, b, c)] == [3, 3, 2]
    s.apply(False, [c, a], [1, 0])                           # 1 raises c; 0 does not lower a
    assert s.info()[0] == 3
    assert [s.lookup(bytes.fromhex(x)) for x in (a, b, c)] == [3, 3, 3]


def test_shared_prefixes_growth_and_absent_ids():
    """Ids sharing their first 16 bytes (a submitter chooses claimed ids), added across several doublings in calls that repeat ids: every
    id is found, 10^5 absent ids are not, and the seeded index keeps probe chains short."""
    rng = np.random.default_rng(11)
    prefix = bytes(16)
    raw = [prefix + bytes(rng.integers(0, 256, 16, dtype=np.uint8)) for _ in range(40000)]
    s = txidutil.HostSet(seed=0x1234)
    s.apply(True, [_hex(raw[0])])
    sizes = []
    for k in range(0, len(raw), 5000):
        chunk = [_hex(x) for x in raw[k:k + 5000]] + [_hex(x) for x in raw[max(0, k - 50):k]]      # repeats of the previous call
        s.apply(False, chunk)
        sizes.append(s.info()[1])
    assert s.info()[0] == len(raw)
    assert sizes[-1] >= 2 * len(raw) and len(set(sizes)) >= 4            # grew across several doublings, load <= 1/2
    assert all(s.lookup(x) == 2 for x in raw)
    absent = 0
    for _ in range(100000):
        x = prefix + bytes(rng.integers(0, 256, 16, dtype=np.uint8))
        absent += s.lookup(x) != 0
    assert absent == 0
    assert s.max_probe() < 64


def test_byte_bound_breaks_the_set_until_replaced():
    ids = [hashlib.sha256(b"%d" % k).hexdigest() for k in range(600)]
    s = txidutil.HostSet(max_bytes=36 * 1024)
    s.apply(True, ids[:400])
    assert s.info() == (400, 1024)
    with pytest.raises(txidutil.SetError, match="FABGPU_TXID_MAX_BYTES") as e:
        s.apply(False, ids[400:])
    assert e.value.failed
    assert s.info()[0] == 0
    assert s.lookup(bytes.fromhex(ids[0])) == 3 and s.lookup(hashlib.sha256(b"absent").digest()) == 3
    with pytest.raises(txidutil.SetError, match="broken"):
        s.apply(False, ids[:1])
    s.apply(True, ids[:10])
    assert s.lookup(bytes.fromhex(ids[0])) == 2 and s.lookup(bytes.fromhex(ids[20])) == 0
    s.apply(True, [])
    assert s.info() == (0, 0) and s.lookup(bytes.fromhex(ids[0])) == -1
