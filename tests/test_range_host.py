"""Range queries in the MVCC stage with an ordered key index (stateindex.cuh, stateset.cuh) on the host build: the written-out cases,
the Merkle helper against hand-built trees, the reference's early-exit hash validator against the final comparison, and generated block
sequences over hot ranges -- each against range_oracle."""
import hashlib

import numpy as np
import pytest

import mvcc_oracle as mo
import range_oracle as ro
import rangecases
import rangeutil


def _run_host(state0, steps):
    s = rangeutil.RangeHost()
    s.replace([(k, v) for k, v in sorted(state0.items())], 1)
    return rangeutil.run_case(state0, steps, s.mvcc, s.update) + (s,)


@pytest.mark.parametrize("case", rangecases.cases(), ids=lambda c: c[0])
def test_case_oracle_and_host_build(case):
    _, state0, steps = case
    out, state, s = _run_host(state0, steps)
    for k, (got, exp, codes) in enumerate(out):
        assert exp == codes, k
        assert got == exp, k
    assert (s.info()[0], s.info()[3]) == mo.info(state)
    for key, v in state.items():
        st, ver = s.lookup(key)
        assert (st == 3) if v == mo.UNKNOWN else (st == 2 and ver == v), key


def _h(b):
    return hashlib.sha256(b).digest()


def _leaf(results):
    return _h(b"".join(ro.pb.f_bytes(1, ro.kv_read(k, v)) for k, v in results))


def test_merkle_helper_against_hand_built_trees():
    res = [(b"k%02d" % i, (1, i)) for i in range(40)]
    d = 3
    # max_degree + 1 results: one leaf, the summary is that leaf at level 1
    assert ro.summary_of(res[:4], d) == ro.Merkle(3, 1, [_leaf(res[:4])])
    # max_degree or fewer: no summary
    assert ro.summary_of(res[:3], d) is None
    # 2 (max_degree + 1) + 1 results: two full leaves and one of a single result
    assert ro.summary_of(res[:9], d) == ro.Merkle(3, 1, [_leaf(res[:4]), _leaf(res[4:8]), _leaf(res[8:9])])
    # 40 results: 10 leaves; level 1 is combined into level 2 whenever it holds max_degree + 1 = 4 hashes, and done() combines the two
    # leftover leaves and carries them up, where level 2 then holds 3 hashes
    lv = [_leaf(res[i:i + 4]) for i in range(0, 40, 4)]
    assert ro.summary_of(res, d) == ro.Merkle(3, 2, [_h(b"".join(lv[0:4])), _h(b"".join(lv[4:8])), _h(b"".join(lv[8:10]))])
    # 53 results: 14 leaves (the last of one result); done() carries level 1 up, level 2 then holds 4 > max_degree and is combined once more
    res2 = res + [(b"z%02d" % i, (2, i)) for i in range(13)]
    lv = [_leaf(res2[i:i + 4]) for i in range(0, 53, 4)]
    l2 = [_h(b"".join(lv[0:4])), _h(b"".join(lv[4:8])), _h(b"".join(lv[8:12])), _h(b"".join(lv[12:14]))]
    assert ro.summary_of(res2, d) == ro.Merkle(3, 3, [_h(b"".join(l2))])
    # a tree that reaches level 3 during update(): max_degree 2, 27 results, 9 leaves of 3
    res3 = [(b"y%03d" % i, (0, i)) for i in range(27)]
    lv = [_leaf(res3[i:i + 3]) for i in range(0, 27, 3)]
    l2 = [_h(b"".join(lv[i:i + 3])) for i in range(0, 9, 3)]
    assert ro.summary_of(res3, 2) == ro.Merkle(2, 3, [_h(b"".join(l2))])
    # and one more result: a leaf of one result at done(), carried from level 1 to 2, then as the only level-2 hash up to level 3
    res4 = res3 + [(b"y999", (0, 0))]
    assert ro.summary_of(res4, 2) == ro.Merkle(2, 3, [_h(b"".join(l2)), _leaf(res4[27:])])


def test_reference_hash_validator_early_exits():
    """The reference's early-exit loop against the final comparison: where it returns, it agrees with Done()'s comparison; it panics
    (index out of range) when the top level rises after lastMatchedIndex passed 0 -- the recorded summary of a prefix of the results."""
    rng = np.random.default_rng(5)
    panics = 0
    for _ in range(600):
        n = int(rng.integers(0, 60))
        res = [(b"k%03d" % i, (int(rng.integers(0, 3)), int(rng.integers(0, 3)))) for i in sorted(rng.choice(300, n, replace=False))]
        d = int(rng.integers(2, 5))
        x = rng.random()
        # the recorded summary: of the results, of a prefix of them (then more results arrive), of a mangled level or hash list
        rec_res = res[: int(rng.integers(0, len(res) + 1))] if x < 0.5 else res
        rec = ro.summary_of(rec_res, d) or ro.Merkle(d, 1, [])
        if x > 0.8 and rec.hashes:
            rec = ro.Merkle(d, rec.max_level + int(rng.integers(-1, 2)), rec.hashes[: int(rng.integers(0, len(rec.hashes) + 1))])
        final = ro.summary_of(res, d)
        try:
            assert ro.hash_validate_reference(res, rec) == (final is not None and final == rec)
        except ro.Panic:
            panics += 1
    assert panics >= 3


def _prefix_merkle_tx(rng, pool, state):
    """a range whose Merkle summary covers only a prefix of its committed results: the early-exit loop's out-of-range case"""
    ks = sorted(pool)
    try:
        res = list(ro.results(state, {}, 0, rangecases.CC, ks[0], "", True))
    except ro.Undetermined:
        return None
    d = 2
    cut = int(rng.integers(3, max(4, len(res) + 1)))
    summ = ro.summary_of(res[:cut], d)
    return [dict(ns=rangecases.CC, ranges=[(ks[0], "", True, summ or ro.Merkle(d, 1, []))])]


def test_generated_blocks_over_hot_ranges():
    rng = np.random.default_rng(17)
    pool = ["k%d" % i for i in range(12)]
    state = {(rangecases.CC, "", k.encode()): (0, int(rng.integers(0, 3))) for k in pool[:8]}
    s = rangeutil.RangeHost(seed=21)
    s.replace(sorted(state.items()), 1)
    seen = {0: 0, 11: 0, 254: 0}
    for b in range(1, 300):
        n = int(rng.integers(1, 12))
        txs = [rangeutil.random_range_tx(rng, pool, state) for _ in range(n)]
        if rng.random() < 0.3:
            txs.append(_prefix_merkle_tx(rng, pool, state))
            n += 1
        tv = [int(rng.choice([0, 0, 0, 0, 0, 0, 254, 10])) for _ in range(n)]
        exp, state, is_open = ro.validate(state, b, txs, tv)
        assert s.mvcc(b, txs, tv) == exp, b
        for t, x in zip(txs, exp):
            if t is not None and t[0].get("ranges") and x in seen:
                seen[x] += 1
        if is_open:
            s.update([], b + 1)
        if b % 5 == 0:
            fix = [(k, (b, 0)) for k, v in state.items() if v == mo.UNKNOWN]
            s.update(fix, b + 1)
            state.update(dict(fix))
        assert (s.info()[0], s.info()[3]) == mo.info(state), b
        live, entries, _ = s.index_info()
        assert live == sum(1 for k in state if k[1] == "") and entries >= live, b
    assert min(seen.values()) > 20, seen


def test_without_an_index_ranges_stay_254():
    s = rangeutil.RangeHost()
    s.replace([((rangecases.CC, "", b"a"), (1, 0))], 1, indexed=False)
    assert s.index_info() == (0, 0, 0)
    assert s.mvcc(1, [rangecases.q("a", "b", [("a", (1, 0))]), rangecases.w("q")], [0, 0]) == [254, 0]


def test_index_counts_growth_and_fold():
    s = rangeutil.RangeHost()
    s.replace([((rangecases.CC, "", b"s%05d" % i), (0, 1)) for i in range(100)] + [((rangecases.CC, "c", b"p"), (0, 1))], 1)
    assert s.index_info()[:2] == (100, 100)
    h = 1
    for blk in range(12):                                              # 12 blocks of 500 new keys: the delta passes 4096 and folds
        txs = [rangecases.w(*["n%02d_%03d_%d" % (blk, t, j) for j in range(5)]) for t in range(100)]
        assert s.mvcc(h, txs, [0] * 100) == [0] * 100
        h += 1
    assert s.index_info()[:2] == (6100, 6100)
    s.update([((rangecases.CC, "", b"s%05d" % i), mo.REMOVE) for i in range(50)], h)
    assert s.index_info()[:2] == (6050, 6100)
    got = s.mvcc(h, [rangecases.q("n11_099", "", [("n11_099_%d" % j, (12, 99)) for j in range(5)] +
                                  [("s%05d" % i, (0, 1)) for i in range(50, 100)])], [0])
    assert got == [0]
