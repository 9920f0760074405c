"""The MVCC stage under CouchDB on the host build (tests/host_sim/couch_host.cpp), and generated JSON values for the key and value
checks: structured random documents and byte-level mutations of them."""
import ctypes
import json
import os
import subprocess
import tempfile

import numpy as np

from util import ROOT
from blockutil import _p
import couch_oracle as co
import mvccutil
import rangeutil

_LIB = None


def lib():
    """built into a temporary directory: the source tree is not written"""
    global _LIB
    if _LIB is None:
        so = os.path.join(tempfile.mkdtemp(prefix="fabgpu_couch_"), "libcouch_host.so")
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-o", so, os.path.join(ROOT, "tests", "host_sim", "couch_host.cpp")])
        L = ctypes.CDLL(so)
        L.ch_new.restype = ctypes.c_void_p
        L.ch_new.argtypes = [ctypes.c_ulonglong]
        L.ch_free.argtypes = [ctypes.c_void_p]
        L.ch_range.restype = ctypes.c_void_p
        L.ch_range.argtypes = [ctypes.c_void_p]
        L.ch_database.argtypes = [ctypes.c_void_p, ctypes.c_int]
        L.ch_apply.restype = ctypes.c_char_p
        L.ch_apply.argtypes = [ctypes.c_void_p, ctypes.c_int] + [ctypes.c_void_p] * 7 + [ctypes.c_size_t, ctypes.c_ulonglong, ctypes.c_size_t,
                                                                                           ctypes.c_ulonglong, ctypes.POINTER(ctypes.c_int)]
        L.ch_mvcc.restype = ctypes.c_char_p
        L.ch_mvcc.argtypes = [ctypes.c_void_p] + [ctypes.c_void_p] * 3 + [ctypes.c_ulonglong, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_size_t,
                                                                         ctypes.c_ulonglong, ctypes.POINTER(ctypes.c_int)]
        L.ch_values.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_size_t, ctypes.c_int, ctypes.c_void_p]
        L.rh_info.argtypes = [ctypes.c_void_p, ctypes.c_void_p]
        L.rh_index_info.argtypes = [ctypes.c_void_p, ctypes.c_void_p]
        L.rh_lookup.argtypes = [ctypes.c_void_p, ctypes.c_char_p, ctypes.c_uint32, ctypes.c_char_p, ctypes.c_uint32, ctypes.c_char_p, ctypes.c_uint32,
                                ctypes.c_void_p]
        _LIB = L
    return _LIB


def block_of(txs):
    """rangeutil.block_of with couch_oracle's encoding"""
    blob, res, ht = b"", [], []
    for tx in txs:
        if tx is None:
            res += [0, 0]; ht.append(1)
            continue
        rw = co.encode(tx)
        res += [len(blob) + 8, len(rw)]; ht.append(3)
        blob += bytes(8) + rw
    return np.frombuffer(blob + bytes(64), np.uint8).copy(), np.array(res or [0], np.uint32), np.array(ht or [0], np.uint8)


def blob_of(values):
    off = np.zeros(len(values) + 1, np.uint32)
    off[1:] = np.cumsum([len(v) for v in values])
    b = np.frombuffer(b"".join(values) + b"\x00", np.uint8).copy()
    return b, off


def host_values(values, path=0):
    """ch_values: the host build's verdict bits of each value (path 0 by length, 1 the one-thread scan, 2 the CTA scan)"""
    b, off = blob_of(values)
    out = np.zeros(max(len(values), 1), np.uint32)
    lib().ch_values(_p(b), _p(off), len(values), path, _p(out))
    return out[:len(values)].tolist()


class CouchHost(rangeutil.RangeHost):
    """RangeHost with the state database switch"""

    def __init__(self, seed=0x5EED, couch=True):
        self.L = lib()
        self.c = ctypes.c_void_p(self.L.ch_new(seed))
        self.h = ctypes.c_void_p(self.L.ch_range(self.c))
        self.database(1 if couch else 0)

    def database(self, kind):
        if self.L.ch_database(self.c, kind) != 0:
            raise mvccutil.StateError("unknown state database kind", False)

    def _apply(self, mode, entries, height, hint=0):
        a = mvccutil.arrays(entries)
        failed = ctypes.c_int(0)
        err = self.L.ch_apply(self.c, mode, *[_p(x) for x in a], len(entries), height, hint, 0, ctypes.byref(failed))
        if err is not None:
            raise mvccutil.StateError(err.decode(), bool(failed.value))

    def mvcc(self, block_num, txs, tv):
        blob, res, ht = block_of(txs)
        tv = np.ascontiguousarray(np.asarray(tv, np.uint8))
        flags = np.zeros(max(len(txs), 1), np.uint8)
        failed = ctypes.c_int(0)
        err = self.L.ch_mvcc(self.c, _p(blob), _p(res), _p(ht), block_num, _p(tv if tv.size else np.zeros(1, np.uint8)), _p(flags), len(txs), 0,
                             ctypes.byref(failed))
        if err is not None:
            raise mvccutil.StateError(err.decode(), bool(failed.value))
        return flags[:len(txs)].tolist()

    def __del__(self):
        try:
            self.L.ch_free(self.c)
        except Exception:
            pass


# ---- generated values --------------------------------------------------------------------------------------------------------------
_NAMES = ["a", "b", "owner", "_id", "_rev", "~version", "_deleted", "x_id", "\\u005fid", "\\u007eversion", "é", "_", "", "\\ud800_x",
          "~versio", "id_"]
_NUMS = ["0", "-0", "1", "-12", "3.25", "1e5", "1E-5", "-0.0e+0", "1.7976931348623157e308", "1.7976931348623159e308", "1e309", "-1e309",
         "1e-400", "1e10000", "0e10000", "123456789012345678901234567890", "0.000000000000000000001e330",
         "1.79769313486231580793728971405303415079934e308", "179769313486231580793728971405303415079934132710037826936173778980444968292764750946649017977587207096330286416692887910946555547851940402630657488671505820681908902000708383676273854845817711531764475730270069855571366959622842914819860834936475292719074168444365510704342711559699508093042880177904174771"]


def _doc(rng, depth):
    x = rng.random()
    if depth > 5 or x < 0.35:
        y = rng.random()
        if y < 0.35:
            return rng.choice(_NUMS)
        if y < 0.7:
            return '"' + rng.choice(["v", "hello", "\\n\\t", "\\u00e9", "\\\\", "\\/", "é", "a b", "\\ud83d\\ude00", "_id"]) + '"'
        return rng.choice(["true", "false", "null"])
    if x < 0.75:
        n = int(rng.integers(0, 5))
        return "{" + ",".join('"%s":%s' % (rng.choice(_NAMES), _doc(rng, depth + 1)) for _ in range(n)) + "}"
    n = int(rng.integers(0, 5))
    return "[" + ",".join(_doc(rng, depth + 1) for _ in range(n)) + "]"


def document(rng):
    """a structured random document, mostly an object at the top, with whitespace now and then"""
    d = _doc(rng, 0) if rng.random() < 0.15 else "{" + ",".join('"%s":%s' % (rng.choice(_NAMES), _doc(rng, 1))
                                                               for _ in range(int(rng.integers(0, 6)))) + "}"
    if rng.random() < 0.2:
        d = d.replace(",", rng.choice([" ,", ", ", "\n,\t", "\r\n,"])).replace(":", rng.choice([" :", ": ", ":\t"]))
    if rng.random() < 0.1:
        d = rng.choice([" ", "\n", "\t"]) + d + rng.choice([" ", "\r\n", ""])
    return d.encode()


_INSERT = [b"{", b"}", b"[", b"]", b",", b":", b'"', b"\\", b"\\u", b"e", b"-", b".", b"0", b"1", b"_", b"\x00", b"\x1f", b"\x80", b"\xff",
           b" ", b"\x0b", b"NaN", b"//", b"\xef\xbb\xbf", b"9" * 30, b"e309"]


def mutate(rng, b):
    """a byte-level mutation: delete, insert, replace or truncate"""
    b = bytearray(b)
    for _ in range(int(rng.integers(1, 4))):
        x = rng.random()
        i = int(rng.integers(0, len(b) + 1))
        if x < 0.3 and b:
            del b[min(i, len(b) - 1)]
        elif x < 0.6:
            b[i:i] = rng.choice(_INSERT)
        elif x < 0.85 and b:
            b[min(i, len(b) - 1)] = int(rng.integers(0, 256))
        else:
            del b[i:]
    return bytes(b)


def corpus(seed, n):
    """n values: documents and mutations of them"""
    rng = np.random.default_rng(seed)
    out = []
    while len(out) < n:
        d = document(rng)
        out.append(d)
        out.append(mutate(rng, d))
    return out[:n]


def json_accepts(b):
    """Python's json module on valid UTF-8 input, NaN and Infinity rejected"""
    def reject(_):
        raise ValueError("constant")
    try:
        json.loads(b.decode("utf-8"), parse_constant=reject)
        return True
    except (ValueError, RecursionError):
        return False
