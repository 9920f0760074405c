import ctypes
import importlib
import os
import subprocess

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def pkg():
    return importlib.import_module("fabric-mod_b200")


def have_gpu():
    try:
        import torch
        return torch.cuda.is_available()
    except Exception:
        return False


def be32(x: int) -> np.ndarray:
    return np.frombuffer(int(x).to_bytes(32, "big"), np.uint8).copy()


def from_be(a) -> int:
    return int.from_bytes(bytes(a), "big")


def hash_to_e32(digest: bytes) -> np.ndarray:
    d = digest[:32]
    return np.frombuffer(b"\x00" * (32 - len(d)) + d, np.uint8).copy()


_HS = None


def hostsim():
    """tests/host_sim/libhostsim.so: the device verify code compiled for the host (test helper, not product)."""
    global _HS
    if _HS is None:
        d = os.path.join(ROOT, "tests", "host_sim")
        so = os.path.join(d, "libhostsim.so")
        src = os.path.join(d, "hostsim.cpp")
        hdrs = [os.path.join(ROOT, "fabric-mod_b200", "csrc", h) for h in ("p256_fe.cuh", "p256_point.cuh", "p256_modinv.cuh", "ecdsa_verify.cuh", "ecdsa_batchaffine.cuh", "fieldops.cuh")]
        if not os.path.exists(so) or any(os.path.getmtime(so) < os.path.getmtime(f) for f in [src] + hdrs):
            # host build of the table would take minutes at the product's 16-bit G windows; the algorithm is window-size generic
            subprocess.check_call(["g++", "-O2", "-std=c++17", "-DFAB_WG=8", "-DFAB_WQ=8", "-DFAB_Q_TWO_LEVEL=1", "-shared", "-fPIC", "-o", so, src])
        _HS = ctypes.CDLL(so)
        _HS.hostsim_gtable.restype = ctypes.c_size_t
    return _HS


def hostsim_verify(qx, qy, e, r, s, cached=False, ba=False, small=False):
    arrs = [np.ascontiguousarray(a, dtype=np.uint8).reshape(-1, 32) for a in (qx, qy, e, r, s)]
    n = arrs[0].shape[0]
    out = np.zeros(n, np.uint8)
    fn = hostsim().hostsim_verify_batch_small if small else hostsim().hostsim_verify_batch_ba if ba else (hostsim().hostsim_verify_batch_cached if cached else hostsim().hostsim_verify_batch)
    fn(*[a.ctypes.data_as(ctypes.c_void_p) for a in arrs], ctypes.c_int(n), out.ctypes.data_as(ctypes.c_void_p))
    return out


def field_op_cases(rnd, n):
    """{op: (a, b, expected)} for every op of fabric-mod_b200/csrc/fieldops.cuh, checked on the device (tests/test_gpu_field.py) and
    on the host build (tests/test_host_sim.py): n random operands plus every pair of edge operands (0, 1, m - 1, 2^255 ...) for the
    products, n random values plus small and structured ones for the inversions.  Expected values are Python integers."""
    from oracle import p256
    P, N, R = p256.P, p256.N, 1 << 256
    rp, rn = pow(R, -1, P), pow(R, -1, N)

    def pairs(mod):
        edge = [0, 1, 2, mod - 1, mod - 2, (1 << 255) % mod, (1 << 224) % mod, (1 << 32) - 1, ((1 << 256) - 1) % mod, (1 << 96) % mod]
        a = [rnd.randrange(mod) for _ in range(n)] + [x for x in edge for _ in edge]
        b = [rnd.randrange(mod) for _ in range(n)] + [y for _ in edge for y in edge]
        return a, b

    def units(mod):
        a = [rnd.randrange(1, mod) for _ in range(n)] + [1, 2, 3, mod - 1, mod - 2, (mod - 1) // 2, 1 << 30, (1 << 30) - 1, 1 << 255] + \
            [rnd.getrandbits(k) or 1 for k in range(1, 256)]
        return a, a

    mul_p = lambda a, b: a * b * rp % P
    table = {0: (pairs(P), mul_p), 1: (pairs(P), lambda a, b: (a + b) % P), 2: (pairs(P), lambda a, b: (a - b) % P),
             3: (pairs(N), lambda a, b: a * b * rn % N),
             4: (units(P), lambda a, b: pow(a, -1, P) * R * R % P), 5: (units(N), lambda a, b: pow(a, -1, N) * R % N),
             6: (units(N), lambda a, b: pow(a, -1, N) * R % N), 7: (pairs(P), lambda a, b: a * a * rp % P),
             8: (units(P), lambda a, b: pow(a, -1, P) * R * R % P), 9: (units(N), lambda a, b: pow(a, -1, N)),
             10: (units(P), lambda a, b: pow(a, -1, P)), 11: (pairs(P), mul_p), 12: (pairs(P), mul_p), 13: (pairs(P), mul_p),
             14: (pairs(P), lambda a, b: a * a * rp % P), 15: (pairs(P), mul_p), 16: (pairs(P), mul_p)}
    return {op: (a, b, [f(x, y) for x, y in zip(a, b)]) for op, ((a, b), f) in table.items()}


def mask_bits(mask_words, n):
    return np.unpackbits(np.asarray(mask_words, dtype="<u4").view(np.uint8), bitorder="little")[:n]
