"""The key-level byte code under AddressSanitizer and UndefinedBehaviorSanitizer: tests/host_sim/blockdev_keylevel_asan.cpp runs the walk
(kl_scan_rwset, kl_lenient, kl_emit), the decide stage and the resolve stage with a key policy table over the wire-mutation corpus, the
Block-level mutants, blocks of metadata writes with a hot key, and write-record overflow."""
import os
import struct
import subprocess

import numpy as np

from tools import blockgen
from util import ROOT
import klcases
import test_key_policies
import wiremut


def _hot_block(net, n_tx, seed):
    """every transaction writes and metadata-writes one key; some also write a collection key and metadata-write it"""
    ns = lambda t: [(blockgen.CHAINCODE, 1, ["hot", "k%d" % (t % 7)], [("collection", ["h%d" % (t % 3)], ["h%d" % (t % 3)] if t % 2 else [], 1)],
                     ["hot"] if t % 5 else [])]
    faults = {3: "nonzero_epoch", 8: "cc_name_mismatch", 11: "bad_creator_sig"}
    return blockgen.build_block(net, n_tx, 3, {t: f for t, f in faults.items() if t < n_tx}, seed=seed, nthreads=2, namespaces=ns)[0]


def test_key_level_code_under_sanitizers(tmp_path):
    d = os.path.join(ROOT, "tests", "host_sim")
    exe = str(tmp_path / "blockdev_keylevel_asan")
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-g", "-fsanitize=address,undefined", "-fno-sanitize-recover=all", "-fno-omit-frame-pointer",
                           "-o", exe, os.path.join(d, "blockdev_keylevel_asan.cpp"), os.path.join(ROOT, "fabric-mod_b200", "csrc", "blockval.cpp")])
    net, ids, _, _, blocks = wiremut.corpus()
    u32 = lambda v: struct.pack("<I", v & 0xffffffff)
    lb = lambda b: u32(len(b)) + bytes(b)
    nodes = np.ascontiguousarray(net.policy_n_of(2), np.int32)
    head = u32(len(ids)) + b"".join(lb(i[0]) + lb(i[1].encode()) + bytes([1 if i[3] else 0]) for i in ids)
    head += u32(nodes.shape[0]) + nodes.tobytes() + u32(len(net.principals)) + b"".join(lb(p.encode()) for p in net.principals) + lb(net.channel.encode())
    kn, r = klcases.vp_forest()
    table = test_key_policies.corpus_key_table(kn, r)
    table[(blockgen.CHAINCODE, "", b"hot")] = r["vp_org1"]
    table[(blockgen.CHAINCODE, "collection", blockgen.key_hash("h1"))] = -2
    kn = np.ascontiguousarray(kn, np.int32)
    enc = lambda x: x.encode() if isinstance(x, str) else bytes(x)
    head += u32(kn.shape[0]) + kn.tobytes() + u32(len(table)) + b"".join(lb(enc(a)) + lb(enc(c)) + lb(enc(k)) + u32(v) for (a, c, k), v in table.items())
    hot = [_hot_block(net, 24, 31), _hot_block(net, 40, 37)]
    items = [(8, b[0]) for b in blocks] + [(8, m) for _, m in wiremut.block_mutants()] + [(8, h) for h in hot] + [(0, hot[0]), (1, hot[1])]
    corpus = tmp_path / "corpus.bin"
    corpus.write_bytes(head + u32(len(items)) + b"".join(u32(h) + u32(16) + lb(b) for h, b in items))
    env = dict(os.environ, ASAN_OPTIONS="detect_leaks=0:halt_on_error=1", UBSAN_OPTIONS="halt_on_error=1:print_stacktrace=1")
    run = subprocess.run([exe, str(corpus)], capture_output=True, text=True, env=env, timeout=900)
    assert run.returncode == 0 and "runtime error" not in run.stderr and "Sanitizer" not in run.stderr, run.stderr[-4000:]
    last = run.stdout.split("\n")[-2].split()
    assert last[:2] == ["blocks", str(len(items))] and int(last[5]) > 3000, last
    assert int(last[7]) > 100 and int(last[9]) > 40, last                      # records made, transactions marked for the resolve stage
    lines = [x for x in run.stdout.split("\n") if x.startswith("flags ")]
    hot_flags = [bytes.fromhex(x.split()[1]) for x in lines[-4:]]
    assert set(hot_flags[2]) <= {254, 3, 25} and {0, 254} <= set(hot_flags[0])   # overflow; an abandoned writer
