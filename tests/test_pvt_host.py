"""The private-data check (pvtdata.cuh) on the host build: every written-out case against its codes and pvt_oracle, and seeded blocks
against pvt_oracle."""
import pytest

import pvt_oracle as po
import pvtcases
import pvtutil


@pytest.mark.parametrize("case", pvtcases.cases(), ids=lambda c: c[0])
def test_case_oracle_and_host_build(case):
    _, txs, flags, pvt, status, verdict = case
    rwsets = pvtcases.rwsets_of(txs, pvt)
    exp = po.validate(rwsets, flags, pvt)
    assert exp == (verdict, status)
    assert pvtutil.host_check(rwsets, flags, pvt) == exp


@pytest.mark.parametrize("seed", range(6))
def test_seeded_blocks_against_the_oracle(seed):
    txs, flags, pvt = pvtcases.seeded(100 + seed, 300)
    rwsets = pvtcases.rwsets_of(txs, pvt)
    got = pvtutil.host_check(rwsets, flags, pvt)
    exp = po.validate(rwsets, flags, pvt)
    assert got == exp
    codes = [s[0] for s in exp[1].values()]
    assert all(codes.count(c) > 0 for c in (po.OK, po.MISMATCH, po.SKIP, po.UNDET)), codes


def test_verdict_follows_the_smallest_deciding_seq():
    """every flag combination of two mismatching entries: the first one flagged VALID or 254 decides"""
    a = pvtcases.kvrwset(5)
    tx = [(pvtcases.CC, [("c1", pvtcases.sha(a))])]
    e = pvtcases.entry([(pvtcases.CC, [("c1", pvtcases.flip(a))])])
    rwsets = pvtcases.rwsets_of([tx, tx])
    for f0 in (0, 254, 11):
        for f1 in (0, 254, 11):
            got = pvtutil.host_check(rwsets, [f0, f1], {0: e, 1: e})
            assert got == po.validate(rwsets, [f0, f1], {0: e, 1: e})
            first = next((s for s, f in enumerate((f0, f1)) if f in (0, 254)), None)
            want = po.OK if first is None else po.MISMATCH if (f0, f1)[first] == 0 else po.UNDET
            assert got[0][0] == want, (f0, f1)
