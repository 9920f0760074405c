"""GPU: the key-table path's scalar preparation (ecdsa_prep_kernel).  One CTA of that kernel shares a single inversion among
FAB_PREP_THREADS signatures; a signature with r or s outside [1, n-1] must contribute 1 to the shared product and come out INVALID
without disturbing its neighbours.  Such signatures sit at the first, a middle and the last position of a CTA's group, among
honest ones, in batches whose size is not a multiple of the CTA width, and every verdict is checked against the oracle."""
import numpy as np
import pytest

from oracle import blockval as ob
from oracle import fast, p256
from tools import blockgen, workload
from tools import fabricpb as pb
from util import be32, from_be, mask_bits, pkg
import blockutil

pytestmark = pytest.mark.gpu

PREP = 128                    # FAB_PREP_THREADS: signatures per shared inversion
N = p256.N
KINDS = (("s", 0), ("s", N), ("r", 0), ("r", N))


@pytest.fixture(scope="module")
def ctx():
    c = pkg().binding.Context(max_batch=8192)
    yield c
    c.close()


def _positions(n):
    """{index: (field, value)}: CTA k of the first four holds kind k at its first, a middle and its last position; the partial
    last CTA holds every kind, its last signature included."""
    bad = {}
    for k, kind in enumerate(KINDS):
        for p in (0, PREP // 2 + k, PREP - 1):
            bad[k * PREP + p] = kind
    tail = 4 * PREP
    for p, kind in zip((tail, tail + 1, (tail + n) // 2, n - 1), KINDS):
        bad[p] = kind
    return bad


def _batch():
    n = 4 * PREP + 77
    w = workload.Workload(n, 8, seed=0x9E9)
    bad = _positions(n)
    for i, (field, v) in bad.items():
        getattr(w, field)[i] = be32(v)
    honest = fast.valid_mask(fast.verify_batch(w.keys_xy, w.key_idx, w.digest, w.dig_off(), w.sigs, w.sig_off, nthreads=8))
    exp = mask_bits(honest, n).astype(bool)
    for i in bad:                                                    # the oracle on the raw tuple (the DER blob still holds the honest one)
        q = w.keys_xy[w.key_idx[i]]
        exp[i] = p256.ecdsa_verify_go114(from_be(q[:32]), from_be(q[32:]), bytes(w.digest[i]), from_be(w.r[i]), from_be(w.s[i]))
    assert not exp[list(bad)].any() and exp.sum() == n - len(bad)
    return w, exp


def test_range_gate_inside_one_shared_inversion_device_resident(ctx):
    import torch
    w, exp = _batch()
    slots = ctx.keys_register(w.keys_xy)
    dev = torch.device("cuda:0")
    t = [torch.from_numpy(np.ascontiguousarray(a)).to(dev) for a in (w.digest, w.r, w.s)]
    ks = torch.from_numpy((slots & 0xFFF)[w.key_idx]).to(dev)
    mask = torch.zeros((w.n + 31) // 32, dtype=torch.int32, device=dev)
    st = torch.cuda.current_stream(dev)
    ctx.verify_p256_device_keyed(True, ks.data_ptr(), 0, 0, t[0].data_ptr(), t[1].data_ptr(), t[2].data_ptr(), w.n, mask.data_ptr(), 0, st.cuda_stream)
    st.synchronize()
    assert (mask_bits(mask.cpu().numpy().view(np.uint32), w.n).astype(bool) == exp).all()


def test_range_gate_inside_one_shared_inversion_pinned_slots(ctx):
    w, exp = _batch()
    slots = ctx.keys_register(w.keys_xy)
    for slot, ks in ((0, slots[w.key_idx]), (1, np.where(w.key_idx % 3 == 0, -1, slots[w.key_idx]))):     # all tabled, then mixed
        hb = ctx.host_buffers(slot)
        for name, arr in (("qx", w.qx()), ("qy", w.qy()), ("e", w.digest), ("r", w.r), ("s", w.s)):
            hb[name][: w.n] = arr
        ctx.host_key_slots(slot)[: w.n] = ks
        ctx.verify_p256_keyed(slot, w.n)
        assert (mask_bits(hb["mask"], w.n).astype(bool) == exp).all(), slot


def test_range_gate_inside_one_shared_inversion_block_path(ctx):
    """Creator signatures with r or s outside [1, n-1] in a block whose job count the device decides (n_dev): r = n passes the DER
    and low-S gates and reaches the prep kernel's range gate; the others stop at the gates.  Creator jobs come first, one per
    transaction, so transaction t is job t of the prep kernel."""
    n_tx = PREP + 45
    bad = {0: ("r", N), PREP // 2: ("r", N), PREP - 1: ("r", N), PREP: ("r", N), n_tx - 1: ("r", N),
           1: ("s", 0), PREP - 2: ("s", N), PREP + 1: ("r", 0)}

    def mutate(t, part, b):
        if part != "Envelope" or t not in bad:
            return b
        env = pb.parse(b, {1: ("payload", "bytes"), 2: ("signature", "bytes")})
        r, s = _der_rs(env["signature"])
        field, v = bad[t]
        r, s = (v, s) if field == "r" else (r, v)
        return pb.envelope(env["payload"], blockgen._der_sig(r, s))

    net = blockgen.Network()
    blk, _ = blockgen.build_block(net, n_tx, 3, {}, seed=61, mutate=mutate)
    ids = blockutil.identities_of(net)
    ctx.msp_configure(ids, net.policy_n_of(3), net.principals, net.channel)
    exp = ob.validate_block(blk, ids, net.channel, net.policy_n_of(3), net.principals, known=[i[0] for i in ids])
    got = ctx.validate_block(blk)
    assert got.tolist() == exp.tolist()
    assert all(exp[t] != ob.VALID for t in bad) and all(exp[t] == ob.VALID for t in range(n_tx) if t not in bad)


def _der_rs(sig):
    """(r, s) of a DER ECDSA-Sig-Value as the signer wrote it (short-form lengths)."""
    assert sig[0] == 0x30
    lr = sig[3]
    r = int.from_bytes(sig[4:4 + lr], "big")
    ls = sig[5 + lr]
    s = int.from_bytes(sig[6 + lr:6 + lr + ls], "big")
    return r, s
