"""GPU: a context that replaces or grows every kind of buffer it owns, checked against the oracle after each step, three times over in
fresh contexts; the device memory the first context gave back stays given back after the third."""
import importlib
import os

import numpy as np
import pytest

from oracle import blockval as ob
from oracle import fast
from tools import blockgen, workload
from util import pkg
import blockutil
import nodeou

pytestmark = pytest.mark.gpu

MAX_BATCH = 8192
SMALL_SLOTS = 20000         # room for one registration of more keys than the 16 384 the build scratch is first sized for
SMALL_KEYS = 16500
LEAK_LIMIT = 256 << 20


def _inputs():
    net = blockgen.Network()
    small, _ = blockgen.build_block(net, 40, 3, {t: blockgen.FAULTS[t % len(blockgen.FAULTS)] for t in range(1, 40, 3)}, seed=5)
    big, _ = blockgen.build_block(net, 10000, 3, {}, seed=17)
    ids = blockutil.identities_of(net)
    blocks = [(blk, ob.validate_block(blk, ids, net.channel, net.policy_n_of(3), net.principals, known=[i[0] for i in ids]).tolist())
              for blk in (small, big)]
    batches = []
    for n, K, seed in ((1500, 8, 31), (6000, 40, 32)):          # both the signature and the key capacities grow
        w = workload.Workload(n, K, seed=seed)
        w.tamper_r(0.05)
        batches.append((w, fast.verify_batch(w.keys_xy, w.key_idx, w.digest, w.dig_off(), w.sigs, w.sig_off, nthreads=8)))
    cases = {c[0]: c for c in nodeou.policy_cases()}
    policies = [nodeou.materialize(cases[name]) for name in ("namespaces_implicit_and_signature_roots", "stock_majority_4_orgs")]
    wp = workload.Workload(3000, 12, seed=33)
    wp.tamper_r(0.05)
    peer_exp = fast.valid_mask(fast.verify_batch(wp.keys_xy, wp.key_idx, wp.digest, wp.dig_off(), wp.sigs, wp.sig_off, nthreads=8))
    ws = workload.Workload(MAX_BATCH, SMALL_KEYS, seed=34)
    ws.tamper_r(0.05)
    small_exp = fast.valid_mask(fast.verify_batch(ws.keys_xy, ws.key_idx, ws.digest, ws.dig_off(), ws.sigs, ws.sig_off, nthreads=8))
    return net, blocks, batches, policies, (wp, peer_exp), (ws, small_exp)


def _one_context(inputs):
    import torch
    sharding = importlib.import_module("fabric-mod_b200.sharding")
    net, blocks, batches, policies, (wp, peer_exp), (ws, small_exp) = inputs
    c = pkg().binding.Context(max_batch=MAX_BATCH)
    try:
        # block slot buffers and the pinned block buffer: a 40-tx block, a 10 k-tx block, the 40-tx block again
        c.msp_configure(blockutil.identities_of(net), net.policy_n_of(3), net.principals, net.channel)
        for blk, exp in (blocks[0], blocks[1], blocks[0]):
            pinned = c.block_buffer(len(blk))
            pinned[:] = np.frombuffer(blk, np.uint8)
            assert c.validate_block(pinned).tolist() == exp
        # the in-place bccsp batch buffers, grown twice
        for w, exp in batches:
            K, n = c.bccsp_fill_batch_buffers(0, w.keys_xy, w.key_idx, w.digest, w.dig_off(), w.sigs, w.sig_off)
            c.bccsp_verify_batch_inplace_async(0, K, n)
            assert (c.bccsp_verify_batch_wait(0, n) == exp).all()
        # the device MSP copy replaced twice, with principal bits, namespace policies and identity groups each time
        for pnet, blk, info, nodes, names, bits, pol, expected in policies:
            c.msp_configure(pnet.identities(), nodes, names, pnet.channel, policies=pol)
            c.msp_principal_bits(bits)
            assert c.validate_block(blk).tolist() == expected
            assert c.validate_envelopes(info["env_blob"], info["env_off"]).tolist() == expected
        # peer-memory mask exchange with one rank: create, open, one step, close
        dev = torch.device("cuda", 0)
        slots = c.keys_register(wp.keys_xy[:8]) & 0xFFF
        slot_of = np.full(wp.K, -1, np.int32)
        slot_of[:8] = slots
        ex = sharding.PeerMaskExchange(c, wp.n, 1, 0, dev)
        assert ex.ok, ex.error
        t = [torch.from_numpy(np.ascontiguousarray(a)).to(dev) for a in (wp.qx(), wp.qy(), wp.digest, wp.r, wp.s, slot_of[wp.key_idx])]
        st = torch.cuda.current_stream(dev)
        full = ex.verify(False, t[5].data_ptr(), t[0].data_ptr(), t[1].data_ptr(), t[2].data_ptr(), t[3].data_ptr(), t[4].data_ptr(), wp.n, st.cuda_stream)
        st.synchronize()
        assert (full.cpu().numpy().view(np.uint32) == peer_exp).all()
        ex.close()
        del t, full
        # one small-table registration of more keys than the build scratch holds
        assert c.small_slot_capacity() > SMALL_KEYS
        hs = c.keys_register_small(ws.keys_xy)
        assert (hs <= -2).all()
        hb = c.host_buffers(0)
        for name, arr in (("qx", ws.qx()), ("qy", ws.qy()), ("e", ws.digest), ("r", ws.r), ("s", ws.s)):
            hb[name][: ws.n] = arr
        c.host_key_slots(0)[: ws.n] = hs[ws.key_idx]
        c.verify_p256_keyed(0, ws.n)
        assert (hb["mask"][: ws.n // 32] == small_exp).all()
    finally:
        c.close()
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    return torch.cuda.mem_get_info()[0]


def test_every_growing_buffer_three_contexts():
    inputs = _inputs()
    saved = {k: os.environ.get(k) for k in ("FABGPU_SMALL_SLOTS", "FABGPU_KEY_SLOTS")}
    os.environ["FABGPU_SMALL_SLOTS"] = str(SMALL_SLOTS)
    os.environ["FABGPU_KEY_SLOTS"] = "64"       # 4 GiB of key tables is enough here; the GPU is shared
    try:
        free = [_one_context(inputs) for _ in range(3)]
    finally:
        for k, v in saved.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v
    drop = free[0] - free[2]
    print("free device memory after each close: %s MiB; after the third %.1f MiB below the first" % ([f >> 20 for f in free], drop / 2**20))
    assert drop <= LEAK_LIMIT, "device memory not given back: %.1f MiB" % (drop / 2**20)
