"""CouchDB cases for the MVCC stage, with their codes written out: (name, state before, steps) as rangecases, in couch_oracle's
transaction form (a write's third element is its value).  The codes are CouchDB's; the same blocks under LevelDB give range_oracle's."""
import rangecases as rc

V, N, I = 0, 254, 24
CC = rc.CC
S = rc.S
A, B = rc.A, rc.B


def wv(key, value, delete=False):
    return [dict(ns=CC, writes=[(key, delete, value)])]


def one_each(values, key="w%d"):
    """one transaction per value, each writing its own key"""
    return [wv(key % i, v) for i, v in enumerate(values)]


RESERVED = [
    (b'{"_id":"x"}', I), (b'{"_rev":"1-abc"}', I), (b'{"_deleted":true}', I), (b'{"_attachments":{}}', I), (b'{"~version":"x"}', I),
    (b'{"\\u005fid":1}', I), (b'{"\\u005Fid":1}', I), (b'{"\\u007eversion":1}', I), (b'{"a":1, "_id":2}', I), (b' {"a":{"_id":1}} ', V),
    (b'{"a":1,"a":2}', V), (b'{"_id":1,"_id":2}', I), (b'{"~versio":1}', V), (b'{"~versions":1}', V), (b'{"x_id":1}', V),
    (b'{"\\ud800_id":1}', V), (b'{"\xff_id":1}', V), (b'{"":1}', V), (b'{"\\u005f":1}', I), (b'{"a":[{"_id":1}]}', V),
]
NOT_OBJECT = [(b'["_id"]', V), (b'"_id"', V), (b'[{"_id":1}]', V), (b'null', V), (b'123', V), (b'true', V), (b' null ', V)]
NOT_JSON = [(b'{"_id":1,}', V), (b'{"_id":1}/*c*/', V), (b'\xef\xbb\xbf{"_id":1}', V), (b'{"_id":NaN}', V), (b'{"_id":1}x', V),
            (b"{'_id':1}", V), (b'{"_id":01}', V), (b'{"_id":"a\tb"}', V), (b'{"_id":1', V), (b'{"_id":1}\x0b', V)]
NUMBERS = [(b'{"_id":1,"n":1.7976931348623157e308}', I), (b'{"_id":1,"n":1.7976931348623159e308}', V), (b'{"_id":1,"n":1e309}', V),
           (b'{"_id":1,"n":1e-400}', I), (b'{"_id":1,"n":[-1e309]}', V), (b'{"_id":1,"n":1.7976931348623158079372897140530341507993e308}', N),
           (b'{"_id":1,"n":1e10000}', N), (b'{"n":1e10000}', V), (b'{"_id":1,"n":0e99999}', I),
           (b'{"_id":1,"n":' + b"17976931348623157" + b"0" * 292 + b"}", I)]


def cases():
    out = []
    for name, vals in (("reserved names", RESERVED), ("non-object tops", NOT_OBJECT), ("not JSON", NOT_JSON), ("numbers", NUMBERS)):
        out.append((name, dict(S), [(one_each([v for v, _ in vals]), [V] * len(vals), [c for _, c in vals])]))
    bad_keys = [b"", b"_a", b"\xff", b"\xed\xa0\x80", b"\xc0\xaf", b"ok\xf4\x90\x80\x80", b"\xe2\x82"]
    good_keys = ["é", "\x00owner\x00alice\x00a1", b"\x7f", "k\U0010ffff"]
    txs = [wv(k, b"value") for k in bad_keys] + [wv(k, False) for k in bad_keys[:2]] + [wv(k, b'{"a":1}') for k in good_keys]
    out.append(("bad and good keys", dict(S), [(txs, [V] * len(txs), [I] * (len(bad_keys) + 2) + [V] * len(good_keys))]))
    out.append(("deletes carrying values", dict(S), [
        ([wv("a", b'{"_id":1}', True), wv("b", b'{"x":1}', True), wv("c", False, True), [dict(ns=CC, reads=[A])]], [V] * 4, [I, V, V, V]),
        ([[dict(ns=CC, reads=[("b", None), ("c", None), A])]], [V], [V])]))
    out.append(("a 24 writer drops out", dict(S), [
        ([wv("a", b'{"_id":1}'), [dict(ns=CC, reads=[A], writes=[("b", False, b'{"v":2}')])], [dict(ns=CC, reads=[("b", (1, 1))])]],
         [V, V, V], [I, V, 11])]))
    out.append(("24 wins over a read conflict and an undecided value", dict(S), [
        ([[dict(ns=CC, reads=[("a", (9, 9))], writes=[("a", False, b'{"_id":1}')])],
          [dict(ns=CC, writes=[("x", False, b'{"_id":1,"n":1e10000}'), ("", False, b"v")])],
          [dict(ns=CC, reads=[("a", (9, 9))], writes=[("y", False, b'{"_id":1,"n":1e10000}')])]], [V, V, V], [I, I, N])]))
    out.append(("validator 254 with a bad write", dict(S), [
        ([wv("a", b'{"_id":1}'), [dict(ns=CC, reads=[A])], wv("d", b'{"_id":1}')], [N, V, 10], [N, N, 10])]))
    out.append(("hashed and metadata writes are not checked", dict(S), [
        ([[dict(ns=CC, md=["_m"], colls=[("coll", [], [(b"\xff" * 32, False)], [])])]], [V], [V])]))
    out.append(("reads and range bounds", dict(S), [
        ([[dict(ns=CC, reads=[("_x", None)])], [dict(ns=CC, reads=[("é", None)])], rc.q(b"\xff", "", []), rc.q("a", b"b\xff", [A]),
          rc.q("a", "_z", [], exhausted=False), rc.q("a", "", [A, B, rc.Cv, rc.D], exhausted=False), rc.q("a", "c", [A, B]),
          rc.q("a", "c", [A, B, rc.Cv], exhausted=False), rc.q(b"\x00", "b", [A])], [V] * 9, [N, V, N, N, N, N, V, V, V])]))
    out.append(("blocks in sequence", dict(S), [
        ([wv("a", b'{"v":1}'), wv("b", b'{"_rev":"x"}'), [dict(ns=CC, reads=[("a", (1, 0))])]], [V, V, V], [V, I, 11]),
        ([[dict(ns=CC, reads=[("a", (1, 0)), B])], wv("n", b'{"_id":1,"n":1.79769313486231580793728971405303415079934e308}')],
         [V, V], [V, N]),
        ([[dict(ns=CC, reads=[("n", (2, 0))])]], [V], [N])]))
    return out
