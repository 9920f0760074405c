"""The MVCC stage under CouchDB (couchval.cuh, stateset.cuh) on the host build: the written-out cases in both modes, the value check on
generated documents and mutations of them against couch_oracle, the oracle's scanner and number rule against Python's json and float,
the key refusals of the install calls, and generated block sequences -- each against couch_oracle."""
import json

import numpy as np
import pytest

import couch_oracle as co
import couchcases
import couchutil
import mvcc_oracle as mo
import mvccutil
import range_oracle as ro
import rangeutil


def _run(state0, steps, couch):
    s = couchutil.CouchHost(couch=couch)
    s.replace(sorted(state0.items()), 1)
    state, height, out = dict(state0), 1, []
    for txs, tv, codes in steps:
        got = s.mvcc(height, txs, tv)
        exp, state, is_open = co.validate(state, height, txs, tv, couch=couch)
        out.append((got, exp, codes))
        if is_open:
            s.update([], height + 1)
        height += 1
    return out, state, s


@pytest.mark.parametrize("case", couchcases.cases(), ids=lambda c: c[0])
def test_case_oracle_and_host_build(case):
    _, state0, steps = case
    out, state, s = _run(state0, steps, True)
    for k, (got, exp, codes) in enumerate(out):
        assert exp == codes, k
        assert got == exp, k
    assert (s.info()[0], s.info()[3]) == mo.info(state)
    for key, v in state.items():
        st, ver = s.lookup(key)
        assert (st == 3) if v == mo.UNKNOWN else (st == 2 and ver == v), key


@pytest.mark.parametrize("case", couchcases.cases(), ids=lambda c: c[0])
def test_case_in_leveldb_mode_gives_the_range_oracle(case):
    _, state0, steps = case
    out, _, _ = _run(state0, steps, False)
    state = dict(state0)
    for height, (txs, tv, _) in enumerate(steps, 1):
        exp, state, _ = ro.validate(state, height, [co._as_range_tx(t) for t in txs], tv)
        assert out[height - 1][0] == exp, height


def test_case_values_one_by_one():
    vals = [v for group in (couchcases.RESERVED, couchcases.NOT_OBJECT, couchcases.NOT_JSON, couchcases.NUMBERS) for v, _ in group]
    codes = [c for group in (couchcases.RESERVED, couchcases.NOT_OBJECT, couchcases.NOT_JSON, couchcases.NUMBERS) for _, c in group]
    want = {0: co.OK, 24: co.INVALID, 254: co.UNDET}
    assert [co.value_code(v) for v in vals] == [want[c] for c in codes]
    assert [co.code_of_bits(b) for b in couchutil.host_values(vals)] == [want[c] for c in codes]


@pytest.mark.parametrize("path", [1, 2], ids=["one_thread", "cta"])
def test_generated_values_against_the_oracle(path):
    """10^5 documents and mutations through each scan, forced: the host build's verdict bits equal the oracle's"""
    vals = couchutil.corpus(1, 100000 if path == 1 else 30000)
    got = couchutil.host_values(vals, path)
    exp = [co.value_bits(v) for v in vals]
    bad = [(v, g, e) for v, g, e in zip(vals, got, exp) if g != e]
    assert not bad, bad[:5]
    codes = [co.code_of_bits(e) for e in exp]
    assert min(codes.count(c) for c in (co.OK, co.INVALID, co.UNDET)) > 20, [codes.count(c) for c in (0, 1, 2)]


def test_the_two_scans_agree_on_long_documents():
    """documents past the length bound (the stage's CTA scan) and the same bytes through the one-thread scan"""
    rng = np.random.default_rng(8)
    vals = []
    for _ in range(60):
        parts = [couchutil.document(rng) for _ in range(int(rng.integers(200, 900)))]
        d = b'{"a":[' + b",".join(parts) + b'],"' + rng.choice([b"_id", b"b", b"~version"]) + b'":1}'
        vals += [d, couchutil.mutate(rng, d)]
    assert sum(len(v) > co.SHORT_MAX for v in vals) > 60
    one, cta, prod = couchutil.host_values(vals, 1), couchutil.host_values(vals, 2), couchutil.host_values(vals, 0)
    assert one == cta == prod == [co.value_bits(v) for v in vals]


def test_oracle_scanner_against_python_json():
    """on every valid-UTF-8 value of the corpus the scanner accepts what json.loads accepts (NaN and Infinity rejected)"""
    n = 0
    for v in couchutil.corpus(2, 30000):
        if not co.utf8_valid(v):
            continue
        n += 1
        assert co.scan_ok(v) == couchutil.json_accepts(v), v
    assert n > 20000


def test_oracle_number_rule_against_float():
    rng = np.random.default_rng(3)
    toks = [b"1.7976931348623157e308", b"1.7976931348623158e308", b"1.797693134862315807937289714053e308", b"1e308", b"9e307", b"1e309",
            b"17976931348623157" + b"0" * 292, b"17976931348623159" + b"0" * 292, b"0." + b"0" * 400 + b"1e709", b"-1e309", b"1e-400"]
    for _ in range(20000):
        m = "".join(rng.choice(list("0123456789"), int(rng.integers(1, 25))))
        m = m.lstrip("0") or "0"
        frac = "".join(rng.choice(list("0123456789"), int(rng.integers(0, 5))))
        e = int(rng.integers(250, 340))
        toks.append(("%s%s%se%d" % (m, "." if frac else "", frac, e - len(m))).encode())
    for t in toks:
        v = co.number_verdict(t)
        if v != co.NUM_UNDET:
            assert (v == co.NUM_ERR) == (abs(float(t)) == float("inf")), t
    assert co.number_verdict(b"1e10000") == co.NUM_UNDET and co.number_verdict(b"0e10000") == 0


def test_keys_refused_on_install_under_couchdb():
    s = couchutil.CouchHost()
    for bad in (b"", b"_a", b"\xff", b"\xed\xa0\x80"):
        with pytest.raises(mvccutil.StateError):
            s.replace([((couchcases.CC, "", bad), (1, 0))], 1)
    s.replace([((couchcases.CC, "", b"ok"), (1, 0)), ((couchcases.CC, "coll", b"\xff" * 32), (1, 1))], 1)
    with pytest.raises(mvccutil.StateError):
        s.update([((couchcases.CC, "", b"_x"), (1, 2))], 1)
    assert s.info()[0] == 2                                     # nothing changed
    s.database(0)
    s.update([((couchcases.CC, "", b"_x"), (1, 2))], 1)         # LevelDB holds any key
    assert s.info()[0] == 3
    with pytest.raises(mvccutil.StateError):
        s.database(2)


def test_unholdable_key_of_a_254_writer_is_settled_by_removal():
    """A transaction the validator leaves at 254 writes "_a": the stage marks it unknown, and a range over it is 254 until the caller
    removes it -- a removal of a key CouchDB cannot hold is accepted, a version for it is not"""
    CC = couchcases.CC
    s = couchutil.CouchHost()
    state = {(CC, "", b"b"): (0, 1)}
    s.replace(sorted(state.items()), 1)
    txs = [couchcases.wv("_a", b'{"v":1}'), couchcases.wv("b", b'{"v":2}')]
    assert s.mvcc(1, txs, [254, 0]) == [254, 0]
    assert s.info()[3] == 1
    rng_tx = couchcases.rc.q("A", "z", [("b", (1, 1))])
    assert s.mvcc(2, [rng_tx], [0]) == [254]
    with pytest.raises(mvccutil.StateError):
        s.update([((CC, "", b"_a"), (1, 0))], 3)
    s.update([((CC, "", b"_a"), mo.REMOVE), ((CC, "", b"b"), (1, 1))], 3)
    assert s.info()[3] == 0
    assert s.mvcc(3, [rng_tx], [0]) == [0]


def _random_tx(rng, pool, state, vals):
    tx = rangeutil.random_range_tx(rng, pool, state, p_range=0.3)
    if tx is None:
        return None
    ns = tx[0]
    ns["writes"] = [(k, d, vals[int(rng.integers(0, len(vals)))] if rng.random() < 0.8 else (not d)) for k, d, *_ in ns.get("writes", ())]
    if rng.random() < 0.05:
        ns.setdefault("reads", []).append(("_x", None))
    return tx


def test_generated_blocks_against_the_oracle():
    rng = np.random.default_rng(11)
    pool = ["k%d" % i for i in range(10)] + ["é%d" % i for i in range(2)]
    vals = couchutil.corpus(4, 400) + [b'{"_id":1}', b'{"a":1}', b'{"~version":1,"n":1e10000}', b"value"]
    state = {(couchcases.CC, "", k.encode()): (0, int(rng.integers(0, 3))) for k in pool[:8]}
    for couch in (True, False):
        s = couchutil.CouchHost(seed=21, couch=couch)
        st = dict(state)
        s.replace(sorted(st.items()), 1)
        seen = {0: 0, 11: 0, 24: 0, 254: 0}
        for b in range(1, 200):
            n = int(rng.integers(1, 12))
            txs = [_random_tx(rng, pool, st, vals) for _ in range(n)]
            tv = [int(rng.choice([0, 0, 0, 0, 0, 254, 10])) for _ in range(n)]
            exp, st, is_open = co.validate(st, b, txs, tv, couch=couch)
            assert s.mvcc(b, txs, tv) == exp, (couch, b)
            for x in exp:
                if x in seen:
                    seen[x] += 1
            if is_open:
                s.update([], b + 1)
            if b % 5 == 0:
                fix = [(k, (b, 0)) for k, v in st.items() if v == mo.UNKNOWN]
                s.update(fix, b + 1)
                st.update(dict(fix))
            assert (s.info()[0], s.info()[3]) == mo.info(st), b
        assert min(seen[c] for c in (0, 11, 254)) > 20 and (seen[24] > 20) == couch, seen


def test_long_and_deep_values():
    long_obj = b'{"a":"' + b"x" * 20000 + b'","_id":1}'
    deep = lambda d, top=b"{": (b'{"k":' * d if top == b"{" else b"[" * d) + b"1" + (b"}" * d if top == b"{" else b"]" * d)
    vals = [long_obj, b"   [" + b"1," * 10000 + b"1]", b" " * 20000 + b"{}", b'"' + b"y" * 20000 + b'"', deep(127), deep(128), deep(129),
            deep(128, b"["), deep(129, b"["), b'{"_id":1,"d":' + deep(200) + b"}", b'{"_id":1,"d":' + deep(126)[:-1] + b"}"]
    assert couchutil.host_values(vals) == [co.value_bits(v) for v in vals]
    assert [co.value_code(v) for v in vals] == [co.INVALID, co.OK, co.OK, co.OK, co.OK, co.OK, co.UNDET, co.OK, co.OK, co.UNDET, co.OK]
    assert couchutil.host_values(vals, 1) == couchutil.host_values(vals, 2)
