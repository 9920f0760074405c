"""The v1.3-mode byte code under AddressSanitizer and UndefinedBehaviorSanitizer: tests/host_sim/blockdev_v13_asan.cpp runs the walk with
dispatch_plan's v1.3 checks, decide_v13 with the namespace versions, the resolve stage and the block's lscc pass, with a key policy
table, over the wire-mutation corpus, the Block-level mutants and seeded v1.3 blocks."""
import os
import struct
import subprocess

import numpy as np

from tools import blockgen
from util import ROOT
import klcases
import test_key_policies
import test_v13_host
import wiremut


def test_v13_code_under_sanitizers(tmp_path):
    d = os.path.join(ROOT, "tests", "host_sim")
    exe = str(tmp_path / "blockdev_v13_asan")
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-g", "-fsanitize=address,undefined", "-fno-sanitize-recover=all", "-fno-omit-frame-pointer",
                           "-o", exe, os.path.join(d, "blockdev_v13_asan.cpp"), os.path.join(ROOT, "fabric-mod_b200", "csrc", "blockval.cpp")])
    net, ids, _, pol, blocks = wiremut.corpus()
    u32 = lambda v: struct.pack("<I", v & 0xffffffff)
    lb = lambda b: u32(len(b)) + bytes(b)
    nodes = np.ascontiguousarray(net.policy_n_of(2), np.int32)
    head = u32(len(ids)) + b"".join(lb(i[0]) + lb(i[1].encode()) + bytes([1 if i[3] else 0]) for i in ids)
    head += u32(nodes.shape[0]) + nodes.tobytes() + u32(len(net.principals)) + b"".join(lb(p.encode()) for p in net.principals) + lb(net.channel.encode())
    kn, r = klcases.vp_forest()
    table = test_key_policies.corpus_key_table(kn, r)
    kn = np.ascontiguousarray(kn, np.int32)
    enc = lambda x: x.encode() if isinstance(x, str) else bytes(x)
    head += u32(kn.shape[0]) + kn.tobytes() + u32(len(table)) + b"".join(lb(enc(a)) + lb(enc(c)) + lb(enc(k)) + u32(v) for (a, c, k), v in table.items())
    ns = {blockgen.CHAINCODE: "1.0", blockgen.STRICT_NAMESPACE: "", "qscc": "1.0", "cscc": "1.0", "lscc": "1.0", "othercc": "2.0"}
    head += u32(len(ns)) + b"".join(lb(n.encode()) + u32(0) + lb(v.encode()) for n, v in sorted(ns.items()))
    ccs = [(blockgen.CHAINCODE, "1.0"), ("lscc", "1.0"), (blockgen.CHAINCODE, "2.0"), ("qscc", "x"), ("escc", "1.0")]
    rand = [blockgen.build_block(net, 10, 2, seed=s, nthreads=2, chaincode=lambda t, s=s: ccs[(t * (s + 1)) % len(ccs)] if t % 3 else ccs[0],
                                 namespaces=lambda t: [(blockgen.CHAINCODE, 1, 1)] + ([("lscc", 0, 1)] if t == 4 else []))[0] for s in range(4)]
    rand += [test_v13_host.random_block(s, n_tx=30)[1] for s in range(2)]      # another network: creators unknown to this table
    items = [(8, b[0]) for b in blocks] + [(8, m) for _, m in wiremut.block_mutants()] + [(8, x) for x in rand] + [(0, rand[1])]
    corpus = tmp_path / "corpus.bin"
    corpus.write_bytes(head + u32(len(items)) + b"".join(u32(h) + u32(16) + lb(b) for h, b in items))
    env = dict(os.environ, ASAN_OPTIONS="detect_leaks=0:halt_on_error=1", UBSAN_OPTIONS="halt_on_error=1:print_stacktrace=1")
    run = subprocess.run([exe, str(corpus)], capture_output=True, text=True, env=env, timeout=900)
    assert run.returncode == 0 and "runtime error" not in run.stderr and "Sanitizer" not in run.stderr, run.stderr[-4000:]
    last = run.stdout.split("\n")[-2].split()
    assert last[:2] == ["blocks", str(len(items))] and int(last[5]) > 3000, last
    assert int(last[7]) >= 1, last                                              # blocks with an lscc invocation
    lines = [x for x in run.stdout.split("\n") if x.startswith("flags ")]
    codes = set(b"".join(bytes.fromhex("".join(x.split()[1:-1])) for x in lines))
    assert {0, 10, 17, 23, 254, 255} <= codes, sorted(codes)
