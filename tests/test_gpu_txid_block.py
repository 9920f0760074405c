"""GPU: fabgpu_committed_txids_add_block -- the ids the block store indexes, extracted from the submitted block and inserted on the device.
Seeded sequences with three blocks in flight, against the sequential oracle (txid_block_oracle) flag for flag; the set it leaves against
the set _add of the oracle's ids leaves; both entry points and the blocking calls; same-slot reuse right after the call; growth from the
smallest table; every refusal and the broken set."""
import os

import numpy as np
import pytest

from oracle import blockval as ob
from tools import blockgen
from tools import fabricpb as pb
from util import pkg
import blockutil
import txid_block_oracle as tbo
import txidblockcases

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ctx():
    c = pkg().binding.Context(max_batch=8192)
    yield c
    c.close()


def _envs(info):
    off = info["env_off"]
    return [bytes(info["env_blob"][off[t]:off[t + 1]]) for t in range(off.shape[0] - 1)]


def _assemble(envs):
    off = np.zeros(len(envs) + 1, np.uint32)
    off[1:] = np.cumsum([len(e) for e in envs])
    return np.frombuffer(b"".join(envs), np.uint8).copy(), off


def _configure(ctx, net):
    B = pkg().binding
    ids = blockutil.identities_of(net)
    ctx.msp_configure(ids, net.policy_n_of(2), net.principals, net.channel)
    ctx.channel_capability(B.CAP_V2_0)
    return ids


def _oracle(net, ids):
    return lambda blk: ob.validate_block(blk, ids, net.channel, net.policy_n_of(2), net.principals, known=[i[0] for i in ids])


def _held_exactly(ctx, table):
    """the set holds exactly the ids of `table`: the count is theirs, and adding them all with kind 0 (which changes no held id's kind)
    adds nothing"""
    held = ctx.committed_txids_info()[0]
    ctx.committed_txids_add(list(table), [0] * len(table))
    return held == len(table) and ctx.committed_txids_info()[0] == held


def _sequence(n_blocks, n_tx, seed):
    """Blocks of fresh transactions plus replays of the blocks 1, 2 and 3 before, and, for a few transactions of the next block, the
    same envelope with tx_id emptied (it indexes the computed id, which is the next block's transaction's id).  [(Block bytes, envelopes)]"""
    net = blockgen.Network()
    fresh = [_envs(blockgen.build_block(net, n_tx, 3, None, seed=seed + k, number=k + 1, nthreads=4)[1]) for k in range(n_blocks)]
    rng = np.random.default_rng(seed)
    out = []
    for k in range(n_blocks):
        envs = list(fresh[k])
        for d in (1, 2, 3):
            if k >= d:
                envs += [fresh[k - d][i] for i in rng.choice(n_tx, 5, replace=False)]
        if k + 1 < n_blocks:
            envs += [txidblockcases.with_txid(fresh[k + 1][i], "") for i in rng.choice(n_tx, 4, replace=False)]
        out.append((pb.block(k + 1, envs), envs))
    return net, out


def _run_pipelined(ctx, blocks, max_tx):
    """submits round-robin over the slots, add_block right after each submit; envelopes entry point on odd blocks"""
    B = pkg().binding
    got = [None] * len(blocks)
    for k, (blk, envs) in enumerate(blocks):
        slot = k % B.SLOTS
        if k >= B.SLOTS:
            got[k - B.SLOTS] = ctx.validate_wait(slot, max_tx).tolist()
        if k % 2:
            ctx.validate_envelopes_async(slot, *_assemble(envs))
        else:
            ctx.validate_block_async(slot, blk)
        ctx.committed_txids_add_block(slot)
    for k in range(max(0, len(blocks) - B.SLOTS), len(blocks)):
        got[k] = ctx.validate_wait(k % B.SLOTS, max_tx).tolist()
    return got


@pytest.mark.parametrize("seed", [31, 57])
def test_sequence_matches_the_sequential_oracle(ctx, seed):
    """Three blocks in flight; replays at distance 1, 2 and 3 are 9, computed-id replays are 9, an id installed with kind 1 stays 254;
    flag for flag the oracle's, and the set afterwards is exactly the oracle's table."""
    net, blocks = _sequence(7, 200, seed)
    ids = _configure(ctx, net)
    kind1 = tbo.indexed_ids(blocks[0][1][:3])
    installed = {"0" * 64: 0, **{i: 1 for i in kind1}}
    ctx.committed_txids(list(installed), list(installed.values()))
    got = _run_pipelined(ctx, blocks, 400)
    exp = [f.tolist() for f in tbo.sequence(_oracle(net, ids), blocks, installed)]
    for k in range(len(blocks)):
        assert got[k] == exp[k], k
    codes = [c for f in exp[1:] for c in f]
    assert codes.count(ob.DUPLICATE_TXID) >= 5 * 3 + 4 * 3 and exp[0][:3] == [ob.NOT_VALIDATED] * 3
    table = tbo.after(installed, [envs for _, envs in blocks])
    assert _held_exactly(ctx, table)
    ctx.committed_txids([])


def test_add_block_equals_add_of_the_oracle_ids(ctx):
    """The cases' envelopes (every id form) as one block: add_block leaves the set _add of the oracle's ids leaves, kinds included (an id
    already held with kind 1 stays 1: a replay of it is 254, not 9)."""
    envs = [e for _, e, _ in txidblockcases.cases()]
    expect = {i for _, _, i in txidblockcases.cases() if i is not None}
    assert set(tbo.indexed_ids(envs)) == expect
    net, blocks = _sequence(2, 20, 71)
    ids = _configure(ctx, net)
    held1 = tbo.indexed_ids([blocks[1][1][0]])
    for blocking in (False, True):
        ctx.committed_txids(held1, [1])
        blob, off = _assemble(envs + blocks[0][1])
        if blocking:
            ctx.validate_envelopes(blob, off)
        else:
            ctx.validate_envelopes_async(0, blob, off)
        ctx.committed_txids_add_block(0)
        if not blocking:
            ctx.validate_wait(0, 200)
        table = tbo.after({held1[0]: 1}, [envs + blocks[0][1]])
        assert _held_exactly(ctx, table)
        flags = ctx.validate_block(blocks[1][0]).tolist()
        assert flags == tbo.sequence(_oracle(net, ids), [(blocks[1][0], [])], table)[0].tolist()
        assert flags[0] == ob.NOT_VALIDATED
    ctx.committed_txids([])


def test_blocking_block_call_on_slot_0(ctx):
    """validate_block then add_block(0): the next block's replays are 9"""
    net, blocks = _sequence(2, 50, 83)
    ids = _configure(ctx, net)
    ctx.committed_txids([], capacity=16)
    ctx.validate_block(blocks[0][0])
    ctx.committed_txids_add_block(0)
    assert ctx.validate_block(blocks[1][0]).tolist() == tbo.sequence(_oracle(net, ids), blocks, {})[1].tolist()
    ctx.committed_txids([])


def test_same_slot_reuse_right_after_add_block(ctx):
    """Large blocks on one slot: submit, add_block, wait, and submit the next block at once -- the next block's copy must not overwrite
    the block add_block is still reading, including when the slot's buffers grow.  The set then holds exactly the blocks' ids."""
    net = blockgen.Network()
    sizes = (8000, 8000, 12000)
    fresh = [_envs(blockgen.build_block(net, n, 3, None, seed=400 + k, number=k + 1, nthreads=8)[1]) for k, n in enumerate(sizes)]
    _configure(ctx, net)
    ctx.committed_txids([], capacity=8)
    rng = np.random.default_rng(5)
    blocks = [fresh[0]]
    for k in (1, 2):
        blocks.append(fresh[k] + [fresh[k - 1][i] for i in rng.choice(len(fresh[k - 1]), 300, replace=False)])
    got = []
    for k, envs in enumerate(blocks):
        ctx.validate_envelopes_async(0, *_assemble(envs))
        ctx.committed_txids_add_block(0)
        got.append(ctx.validate_wait(0, 20000).tolist())
    for k, envs in enumerate(blocks):
        exp = [ob.VALID] * len(fresh[k]) + [ob.DUPLICATE_TXID] * (len(envs) - len(fresh[k]))
        assert got[k] == exp, k
    assert _held_exactly(ctx, tbo.after({}, blocks))
    ctx.committed_txids([])


def test_growth_from_a_small_table(ctx):
    """From the smallest table, many blocks through add_block: the table doubles several times while blocks are in flight"""
    B = pkg().binding
    net = blockgen.Network()
    fresh = [_envs(blockgen.build_block(net, 1500, 3, None, seed=600 + k, number=k + 1, nthreads=8)[1]) for k in range(8)]
    _configure(ctx, net)
    ctx.committed_txids(["0" * 64])
    assert ctx.committed_txids_info() == (1, 1024)
    blocks = [(None, envs + (fresh[k - 2][:100] if k >= 2 else [])) for k, envs in enumerate(fresh)]
    sizes = []
    for k, (_, envs) in enumerate(blocks):
        slot = k % B.SLOTS
        if k >= B.SLOTS:
            ctx.validate_wait(slot, 2000)
        ctx.validate_envelopes_async(slot, *_assemble(envs))
        ctx.committed_txids_add_block(slot)
        sizes.append(ctx.committed_txids_info())
    for k in range(len(blocks) - B.SLOTS, len(blocks)):
        flags = ctx.validate_wait(k % B.SLOTS, 2000).tolist()
        assert flags == [ob.VALID] * 1500 + [ob.DUPLICATE_TXID] * 100
    assert len({s[1] for s in sizes}) >= 3
    assert _held_exactly(ctx, tbo.after({"0" * 64: 0}, [envs for _, envs in blocks]))
    ctx.committed_txids([])


def test_refusals_and_broken_set(ctx):
    """No set; a slot with no submitted block; a block added twice; a broken set: FABGPU_E_ARG and nothing changes"""
    B = pkg().binding
    net, blocks = _sequence(2, 30, 97)
    ids = _configure(ctx, net)
    fresh = B.Context(max_batch=8192)
    try:
        _configure(fresh, net)
        fresh.committed_txids(["0" * 64])
        with pytest.raises(B.FabGpuError, match="no submitted block"):
            fresh.committed_txids_add_block(1)
        fresh.committed_txids([])
        fresh.validate_block_async(1, blocks[0][0])
        with pytest.raises(B.FabGpuError, match="no committed tx-id set"):
            fresh.committed_txids_add_block(1)
        fresh.validate_wait(1, 100)
    finally:
        fresh.close()
    with pytest.raises(B.FabGpuError):
        ctx.committed_txids_add_block(B.SLOTS)
    ctx.committed_txids(["0" * 64])
    ctx.validate_block_async(2, blocks[0][0])
    ctx.committed_txids_add_block(2)
    with pytest.raises(B.FabGpuError, match="already added"):
        ctx.committed_txids_add_block(2)
    ctx.validate_wait(2, 100)
    with pytest.raises(B.FabGpuError, match="already added"):
        ctx.committed_txids_add_block(2)
    assert ctx.committed_txids_info()[0] == 1 + len(tbo.indexed_ids(blocks[0][1]))
    saved = os.environ.get("FABGPU_TXID_MAX_BYTES")
    os.environ["FABGPU_TXID_MAX_BYTES"] = str(36 * 1024)
    try:
        with pytest.raises(B.FabGpuError, match="FABGPU_TXID_MAX_BYTES"):
            ctx.committed_txids_add(["%064x" % k for k in range(1000)])
        ctx.validate_block_async(2, blocks[1][0])
        with pytest.raises(B.FabGpuError, match="broken"):
            ctx.committed_txids_add_block(2)
        broken = ctx.validate_wait(2, 100).tolist()
        reaches = tbo.sequence(_oracle(net, ids), [(blocks[1][0], [])], {i: 1 for i in tbo.indexed_ids(blocks[1][1])})[0].tolist()
        assert broken == reaches
        ctx.committed_txids([])
    finally:
        if saved is None:
            os.environ.pop("FABGPU_TXID_MAX_BYTES", None)
        else:
            os.environ["FABGPU_TXID_MAX_BYTES"] = saved
    ctx.committed_txids(["0" * 64])
    ctx.validate_block_async(0, blocks[0][0])
    ctx.committed_txids_add_block(0)
    ctx.validate_wait(0, 100)
    ctx.committed_txids([])
