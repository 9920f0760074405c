"""GPU: contexts of one table group (fabgpu_init_shared) -- three channel contexts validating concurrently against their own oracles,
handles and tables shared through the group, window and small tables recycled across contexts while blocks and batches are in flight,
and a group that outlives the context that made it and gives its memory back with the last one."""
import os
import threading

import numpy as np
import pytest

from oracle import blockval as ob
from oracle import fast
from tools import blockgen, workload
from util import from_be, pkg
import blockutil
import mvcc_oracle as mo
import mvccutil
import tablecheck as tc
import txid_block_oracle as tbo
import v13_oracle

pytestmark = pytest.mark.gpu

MAX_BATCH = 8192
CC = blockgen.CHAINCODE
# faults that leave the read/write set reachable, so the MVCC stage still enumerates the transaction (as in test_gpu_mvcc)
FAULTS = ("bad_creator_sig", "bad_endorsement_sig", "dup_endorser", "unknown_endorser", "unknown_creator", "invalid_creator_cert",
          "high_s_endorsement", "two_bad_endorsements", "dup_txid", "bad_proposal_hash", "many_endorsements")
FAULTS_ONE_ORG = ("bad_creator_sig", "bad_endorsement_sig", "unknown_endorser", "unknown_creator", "invalid_creator_cert",
                  "high_s_endorsement", "dup_txid", "bad_proposal_hash")
assert set(FAULTS) <= set(blockgen.FAULTS)


def _envs(info):
    off = info["env_off"]
    return [bytes(info["env_blob"][off[t]:off[t + 1]]) for t in range(off.shape[0] - 1)]


def _context(**kw):
    return pkg().binding.Context(max_batch=MAX_BATCH, **kw)


def _run_threads(fns):
    errors = []

    def wrap(fn):
        try:
            fn()
        except BaseException as e:           # reported on the main thread
            errors.append(e)

    th = [threading.Thread(target=wrap, args=(fn,)) for fn in fns]
    for t in th:
        t.start()
    for t in th:
        t.join()
    if errors:
        raise errors[0]


class _Channel:
    """A channel: its network, blocks with read/write sets and faults, the validator flags its oracle gives (ledger check included when
    it has a tx-id set), and the world state its table starts from."""

    def __init__(self, net, v13, txids, n_blocks, seed, state_versions):
        self.net, self.v13, self.txids = net, v13, txids
        self.ids = blockutil.identities_of(net)
        rng = np.random.default_rng(seed)
        pool = ["hot%d" % i for i in range(10)]
        self.state0 = {(CC, "", ("hot%d" % i).encode()): state_versions[i] for i in range(len(state_versions))}
        self.blocks = []
        for b in range(n_blocks):
            n = int(rng.integers(12, 28))
            txs = [mvccutil.random_tx(rng, pool, ns_name=CC, unreached=0.0) for _ in range(n)]
            faults = {t: FAULTS[int(rng.integers(len(FAULTS)))] for t in range(n) if rng.random() < 0.15}
            hook = lambda t, part, data, txs=txs: mo.encode(txs[t]) if part == "TxReadWriteSet" else data
            blk, info = blockgen.build_block(net, n, 3, faults, seed=seed * 100 + b, number=b + 1, mutate=hook)
            self.blocks.append((txs, blk, _envs(info)))
        if v13:
            oracle_fn = lambda blk: v13_oracle.validate_block(blk, self.ids, net.channel, net.policy_n_of(3), net.principals,
                                                              policies={CC: 0}, versions={CC: "1.0"}, known=[i[0] for i in self.ids])
        else:
            oracle_fn = lambda blk: ob.validate_block(blk, self.ids, net.channel, net.policy_n_of(3), net.principals,
                                                      known=[i[0] for i in self.ids])
        if txids:
            self.tv = [f.tolist() for f in tbo.sequence(oracle_fn, [(blk, envs) for _, blk, envs in self.blocks], {})]
        else:
            self.tv = [oracle_fn(blk).tolist() for _, blk, _ in self.blocks]

    def configure(self, c):
        B = pkg().binding
        c.msp_configure(self.ids, self.net.policy_n_of(3), self.net.principals, self.net.channel, policies={CC: 0})
        if self.v13:
            c.namespace_versions({CC: "1.0"})
        c.channel_capability(B.CAP_V1_3 if self.v13 else B.CAP_V2_0)
        if self.txids:
            c.committed_txids([], capacity=1024)
        c.state_versions([((k[0], k[1], k[2]), v) for k, v in mvccutil.state_entries(self.state0)], 1)

    def run(self, c):
        """Three blocks in flight; each block's tx ids go into the set right after its submit, its MVCC stage runs after its wait.
        Returns [(validator flags, MVCC flags, expected MVCC flags)] per block."""
        S = pkg().binding.SLOTS
        state, out = dict(self.state0), []

        def submit(k):
            c.validate_block_async(k % S, self.blocks[k][1])
            if self.txids:
                c.committed_txids_add_block(k % S)

        for k in range(min(S, len(self.blocks))):
            submit(k)
        for k, (txs, _, _) in enumerate(self.blocks):
            tv = c.validate_wait(k % S, len(txs) + 16)
            got = c.validate_mvcc(k % S, 1 + k, tv).tolist()
            exp, state, is_open = mo.validate(state, 1 + k, txs, tv.tolist())
            if is_open:
                c.state_versions_update([], 2 + k)
            out.append((tv.tolist(), got, exp))
            if k + S < len(self.blocks):
                submit(k + S)
        return out


def test_three_channels_concurrently():
    """Channels A and B have the same endorsers (one network seed, two channel names) and the same block seeds, so the same tx ids;
    channel C has other endorsers and runs as a V1_3 channel with a state table only.  Three host threads, three blocks in flight each:
    every validator flag array equals its channel's oracle and every MVCC flag array the MVCC oracle over it, so no channel's tx ids,
    state or policies reached another's flags."""
    A = _Channel(blockgen.Network(channel="channel-a"), False, True, 8, 41, [(0, i % 3) for i in range(6)])
    Bc = _Channel(blockgen.Network(channel="channel-b"), False, True, 8, 41, [(1, i % 2) for i in range(8)])
    C = _Channel(blockgen.Network(seed=0xC0FFEE, channel="channel-c"), True, False, 8, 43, [(0, 0) for i in range(4)])
    assert A.blocks[0][2] != Bc.blocks[0][2]
    assert tbo.indexed_ids(A.blocks[0][2]) == tbo.indexed_ids(Bc.blocks[0][2])       # the same ids in both channels
    assert any(ob.DUPLICATE_TXID in f for f in A.tv)
    parent = _context()
    ca, cb = _context(share_tables_with=parent), _context(share_tables_with=parent)
    try:
        chans = ((A, parent), (Bc, ca), (C, cb))
        for ch, c in chans:
            ch.configure(c)
        results = [None] * 3

        def job(i):
            ch, c = chans[i]
            results[i] = ch.run(c)
        _run_threads([lambda i=i: job(i) for i in range(3)])
        moved = 0
        for (ch, _), res in zip(chans, results):
            for k, (tv, got, exp) in enumerate(res):
                assert tv == ch.tv[k], (ch.net.channel, k)
                assert got == exp, (ch.net.channel, k)
                moved += sum(1 for x, y in zip(got, tv) if x != y)
        assert moved > 0                      # the MVCC stage changed flags
        # the tx-id sets hold their own channel's ids: A's and B's are the same ids, C has none
        assert parent.committed_txids_info()[0] == ca.committed_txids_info()[0] > 0
    finally:
        for c in (ca, cb, parent):
            c.close()


def test_handles_and_tables_are_the_groups():
    """Keys registered through the parent have the same handles through a child and build nothing new; the child reads the parent's
    tables (a small table whole and window 0 of a window table, checked on the CPU with the group law); a channel whose endorsers another
    channel of the group already registered builds no window table."""
    B = pkg().binding
    parent = _context()
    child = _context(share_tables_with=parent)
    grandchild = _context(share_tables_with=child)
    try:
        assert child.key_slot_capacity() == parent.key_slot_capacity() == grandchild.key_slot_capacity()
        assert child.small_slot_capacity() == parent.small_slot_capacity()
        w = workload.Workload(64, 6, seed=0x5A1E)
        big, small = w.keys_xy[:3], w.keys_xy[3:]
        hb = parent.keys_register(big)
        hs = parent.keys_register_small(small)
        stats = parent.key_table_stats()
        launches = child.launch_count()
        assert (child.keys_register(big) == hb).all() and (grandchild.keys_register(big) == hb).all()
        assert (child.keys_register_small(small) == hs).all()
        assert child.key_table_stats() == stats == parent.key_table_stats()
        assert child.launch_count() == launches                                  # nothing was built
        # the parent-built tables read through the child
        ws, windows, _ = B.Context.small_table_info()
        per = 1 << (ws - 1)
        window, digit = np.repeat(np.arange(windows), per), np.tile(np.arange(1, per + 1), windows)
        for h, k in zip(hs[:2], small[:2]):
            q = (from_be(k[:32]), from_be(k[32:]))
            rows = child.test_table_entries(int(h), window, digit).tobytes()
            assert tc.check_table(rows, ws, True, q) == []
        wq = B.build_info()[1]
        perq = (1 << wq) - 1
        q = (from_be(big[0][:32]), from_be(big[0][32:]))
        bases = tc.window_bases(q, wq, (256 + wq - 1) // wq)
        rows = child.test_table_entries(int(hb[0]) & 0xFFF, np.zeros(perq, np.uint32), np.arange(1, perq + 1)).tobytes()
        assert tc.check_runs(tc.table_runs(rows, wq, False, bases[:1])) == []
        g = child.test_table_entries(-1, np.zeros(4, np.uint32), np.arange(1, 5)).tobytes()
        assert g == parent.test_table_entries(-1, np.zeros(4, np.uint32), np.arange(1, 5)).tobytes()
        # channel B after channel A, same endorsers: no new window table
        na, nb = blockgen.Network(channel="channel-a"), blockgen.Network(channel="channel-b")
        peers_a = np.stack([np.frombuffer(p.xy, np.uint8) for p in na.peers])
        cap = parent.key_slot_capacity()
        if len(na.msp_table) > cap:
            pytest.skip("the MSP does not fit the window-table pool")
        child.msp_configure(blockutil.identities_of(na), na.policy_n_of(3), na.principals, na.channel)
        before = parent.key_table_stats()
        grandchild.msp_configure(blockutil.identities_of(nb), nb.policy_n_of(3), nb.principals, nb.channel)
        assert parent.key_table_stats()["big"] == before["big"]
        assert (parent.keys_register(peers_a) >= 0).all() and parent.key_table_stats() == before
        blk, _ = blockgen.build_block(nb, 40, 3, {t: FAULTS[t % len(FAULTS)] for t in range(1, 40, 3)}, seed=5)
        ids = blockutil.identities_of(nb)
        exp = ob.validate_block(blk, ids, nb.channel, nb.policy_n_of(3), nb.principals, known=[i[0] for i in ids]).tolist()
        assert grandchild.validate_block(blk).tolist() == exp
    finally:
        for c in (grandchild, child, parent):
            c.close()


def _with_env(env, fn):
    saved = {k: os.environ.get(k) for k in env}
    os.environ.update({k: str(v) for k, v in env.items()})
    try:
        return fn()
    finally:
        for k, v in saved.items():
            if v is None:
                del os.environ[k]
            else:
                os.environ[k] = v


def test_recycling_across_contexts_with_work_in_flight():
    """Four window-table slots and 24 small ones for the group.  Two channels whose MSPs need three window tables each validate blocks
    three deep from their own threads while a third thread verifies batches on the parent with fresh keys (three busy keys per batch take
    window tables, sixteen recurring ones small tables): every registration recycles tables another context's MSP or batch uses.  Every
    flag and status equals the oracle's."""
    parent = _with_env({"FABGPU_KEY_SLOTS": 4, "FABGPU_SMALL_SLOTS": 24}, _context)
    chans = []
    try:
        assert parent.key_slot_capacity() == 4 and parent.small_slot_capacity() == 24
        for seed, name in ((0xA1, "channel-x"), (0xB2, "channel-y")):
            net = blockgen.Network(n_orgs=1, n_clients=1, seed=seed, channel=name)
            ids = blockutil.identities_of(net)
            assert len(ids) <= 4
            blocks = []
            for b in range(6):
                faults = {t: FAULTS_ONE_ORG[(t + b) % len(FAULTS_ONE_ORG)] for t in range(1, 60, 4)}
                blk, _ = blockgen.build_block(net, 60, 1, faults, seed=seed + b, number=b + 1)
                blocks.append((blk, ob.validate_block(blk, ids, net.channel, net.policy_n_of(1), net.principals, known=[i[0] for i in ids]).tolist()))
            c = _context(share_tables_with=parent)
            c.msp_configure(ids, net.policy_n_of(1), net.principals, net.channel)
            chans.append((c, blocks))
        # keys 0..2 carry 1000 signatures each (window tables), keys 3..18 128 each (small tables); fresh keys in every batch
        key_idx = np.random.default_rng(7).permutation(np.concatenate([np.repeat(np.arange(3), 1000), np.repeat(np.arange(3, 19), 128)]))
        batches = []
        for s in range(6):
            w = workload.Workload(key_idx.size, 19, seed=0xF00 + s, key_idx=key_idx)
            w.tamper_r(0.05)
            batches.append(w)
        results = {}

        def run_channel(i):
            c, blocks = chans[i]
            S = pkg().binding.SLOTS
            got = [None] * len(blocks)
            for k in range(min(S, len(blocks))):
                c.validate_block_async(k % S, blocks[k][0])
            for k in range(len(blocks)):
                got[k] = c.validate_wait(k % S, 128).tolist()
                if k + S < len(blocks):
                    c.validate_block_async(k % S, blocks[k + S][0])
            results[i] = got

        def run_batches():
            results["b"] = [parent.bccsp_verify_batch(w.keys_xy, w.key_idx, w.digest, w.dig_off(), w.sigs, w.sig_off) for w in batches]
        _run_threads([lambda: run_channel(0), lambda: run_channel(1), run_batches])
        for i, (c, blocks) in enumerate(chans):
            for k, (_, exp) in enumerate(blocks):
                assert results[i][k] == exp, (i, k)
        for w, st in zip(batches, results["b"]):
            exp = fast.verify_batch(w.keys_xy, w.key_idx, w.digest, w.dig_off(), w.sigs, w.sig_off, nthreads=8)
            assert (st == exp).all()
        stats = parent.key_table_stats()
        assert stats["big"] <= 4 and stats["small_recycled"] > 0
    finally:
        for c, _ in chans:
            c.close()
        parent.close()


def test_child_outlives_parent_and_memory_comes_back():
    """A shared context costs far less device memory than the generator table alone; the child keeps validating blocks and verifying
    batches after the parent is destroyed; once the last context of the group is gone, the memory is back."""
    import torch
    torch.cuda.init()
    free0 = torch.cuda.mem_get_info(0)[0]
    parent = _context()
    free1 = torch.cuda.mem_get_info(0)[0]
    child = _context(share_tables_with=parent)
    free2 = torch.cuda.mem_get_info(0)[0]
    try:
        assert free0 - free1 > (3 << 30)                        # the group's tables
        assert free1 - free2 < (512 << 20), free1 - free2
        net = blockgen.Network()
        ids = blockutil.identities_of(net)
        child.msp_configure(ids, net.policy_n_of(3), net.principals, net.channel)
        blk, _ = blockgen.build_block(net, 200, 3, {t: FAULTS[t % len(FAULTS)] for t in range(1, 200, 5)}, seed=9)
        exp = ob.validate_block(blk, ids, net.channel, net.policy_n_of(3), net.principals, known=[i[0] for i in ids]).tolist()
        w = workload.Workload(4096, 10, seed=0x11FE)
        w.tamper_r(0.05)
        exp_st = fast.verify_batch(w.keys_xy, w.key_idx, w.digest, w.dig_off(), w.sigs, w.sig_off, nthreads=8)
        assert child.validate_block(blk).tolist() == exp
        parent.close()
        assert child.validate_block(blk).tolist() == exp
        assert (child.bccsp_verify_batch(w.keys_xy, w.key_idx, w.digest, w.dig_off(), w.sigs, w.sig_off) == exp_st).all()
        child.keys_register(w.keys_xy[:2])
        assert (child.bccsp_verify_batch(w.keys_xy, w.key_idx, w.digest, w.dig_off(), w.sigs, w.sig_off) == exp_st).all()
    finally:
        child.close()
        parent.close()
    free3 = torch.cuda.mem_get_info(0)[0]
    assert free3 > free0 - (256 << 20), (free0, free3)
