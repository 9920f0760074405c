"""The MVCC stage (stateset.cuh) on the host build: the written-out cases, random blocks over a small hot key pool, the table's refusals,
unknown keys, open blocks, growth and the byte bound -- each against mvcc_oracle."""
import numpy as np
import pytest

import mvcc_oracle as mo
import mvcccases
import mvccutil


def _run_host(state0, blocks):
    s = mvccutil.HostState()
    s.replace(mvccutil.state_entries(state0), 1)
    out = []
    for k, (txs, tv, _) in enumerate(blocks):
        out.append(s.mvcc(1 + k, txs, tv))
        if s.info()[2] != 2 + k:                                      # an open block: close it as a peer would after committing
            s.update([], 2 + k)
    return out, s


@pytest.mark.parametrize("case", mvcccases.cases(), ids=lambda c: c[0])
def test_case_oracle_and_host_build(case):
    _, state0, blocks = case
    state = dict(state0)
    exp = []
    for k, (txs, tv, codes) in enumerate(blocks):
        flags, state, _ = mo.validate(state, 1 + k, txs, tv)
        assert flags == codes
        exp.append(flags)
    host, s = _run_host(state0, blocks)
    assert host == exp
    assert s.info()[0] == mo.info(state)[0] and s.info()[3] == mo.info(state)[1]
    for key, v in state.items():
        st, ver = s.lookup(key)
        assert (st == 3) if v == mo.UNKNOWN else (st == 2 and ver == v), key


def test_random_blocks_over_a_hot_key_pool():
    rng = np.random.default_rng(7)
    pool = ["k%d" % i for i in range(12)]
    state = {(mvcccases.CC, "", k.encode()): (0, int(rng.integers(0, 3))) for k in pool[:8]}
    s = mvccutil.HostState(seed=99)
    s.replace(mvccutil.state_entries(state), 1)
    moved = 0
    for b in range(1, 400):
        n = int(rng.integers(1, 12))
        txs = [mvccutil.random_tx(rng, pool) for _ in range(n)]
        tv = [int(rng.choice([0, 0, 0, 0, 254, 10])) for _ in range(n)]
        exp, state, is_open = mo.validate(state, b, txs, tv)
        assert s.mvcc(b, txs, tv) == exp, b
        moved += sum(1 for x, y in zip(exp, tv) if x != y)
        assert s.info()[2] == (b if is_open else b + 1)
        if is_open:
            s.update([], b + 1)
        if b % 50 == 0:                                              # a peer re-reads the unknown keys from its state database
            fix = [(k, (b, 0)) for k, v in state.items() if v == mo.UNKNOWN]
            s.update(fix, b + 1)
            state.update({k: v for k, v in fix})
        assert (s.info()[0], s.info()[3]) == mo.info(state), b
    assert moved > 300


def test_refusals_keep_the_table():
    s = mvccutil.HostState()
    with pytest.raises(mvccutil.StateError, match="no state version table"):
        s.mvcc(0, [], [])
    key = (mvcccases.CC, "", b"a")
    s.replace([(key, (3, 1))], 5)
    with pytest.raises(mvccutil.StateError, match="height"):
        s.mvcc(4, [mvcccases.r(("a", (3, 1)))], [0])
    with pytest.raises(mvccutil.StateError, match="twice"):
        s.update([(key, (1, 1)), (key, (2, 2))], 5)
    with pytest.raises(mvccutil.StateError, match="below"):
        s.update([(key, (1, 1))], 4)
    assert s.info()[:3] == (1, 1024, 5) and s.lookup(key) == (2, (3, 1))
    assert s.mvcc(5, [None, mvcccases.r(("a", (3, 1)))], [0, 0]) == [254, 254]
    with pytest.raises(mvccutil.StateError, match="open"):
        s.mvcc(5, [], [])
    s.update([(key, mo.REMOVE)], 6)                                   # closes block 5 and removes the key
    assert s.info()[:3] == (0, 1024, 6) and s.lookup(key)[0] == 0
    assert s.mvcc(6, [mvcccases.r(("a", None))], [0]) == [0]


def test_growth_past_half_load_and_removed_keys():
    s = mvccutil.HostState()
    s.replace([((mvcccases.CC, "", b"s%d" % i), (0, i)) for i in range(500)], 1)
    assert s.info()[1] == 1024
    txs = [mvcccases.w(*["n%d_%d" % (t, j) for j in range(4)]) for t in range(10)]
    assert s.mvcc(1, txs, [0] * 10) == [0] * 10
    assert s.info()[:3] == (540, 2048, 2)
    assert s.lookup((mvcccases.CC, "", b"n3_2")) == (2, (1, 3))
    s.update([((mvcccases.CC, "", b"s%d" % i), mo.REMOVE) for i in range(500)], 2)
    assert s.info()[0] == 40 and all(s.lookup((mvcccases.CC, "", b"s%d" % i))[0] == 0 for i in range(500))


def test_byte_bound_breaks_the_table_until_replaced():
    s = mvccutil.HostState(max_bytes=56 * 1024)
    s.replace([((mvcccases.CC, "", b"s%d" % i), (0, 0)) for i in range(500)], 1)
    with pytest.raises(mvccutil.StateError, match="FABGPU_STATE_MAX_BYTES") as e:
        s.update([((mvcccases.CC, "", b"t%d" % i), (0, 0)) for i in range(100)], 1)
    assert e.value.failed and s.info()[0] == 0
    assert s.mvcc(1, [mvcccases.r(("s1", (0, 0))), mvcccases.r(("q", None))], [0, 10]) == [254, 10]
    with pytest.raises(mvccutil.StateError, match="broken"):
        s.update([], 2)
    s.replace([((mvcccases.CC, "", b"s1"), (0, 0))], 1)
    assert s.mvcc(1, [mvcccases.r(("s1", (0, 0)))], [0]) == [0]


def test_unknown_keys_until_update():
    """A 254 writer leaves its keys unknown: a later block's read of one is 254 until _update gives it a version or removes it."""
    s = mvccutil.HostState()
    u, v = (mvcccases.CC, "", b"u"), (mvcccases.CC, "", b"v")
    s.replace([(v, (0, 1))], 1)
    assert s.mvcc(1, [mvcccases.w("u", "v")], [254]) == [254]
    assert s.info() == (2, 1024, 2, 2) and s.lookup(u)[0] == 3
    assert s.mvcc(2, [mvcccases.r(("u", None)), mvcccases.r(("v", (0, 1)))], [0, 0]) == [254, 254]
    s.update([(u, (1, 0)), (v, mo.REMOVE)], 3)
    assert s.info() == (1, 1024, 3, 0)
    assert s.mvcc(3, [mvcccases.r(("u", (1, 0))), mvcccases.r(("v", None))], [0, 0]) == [0, 0]
