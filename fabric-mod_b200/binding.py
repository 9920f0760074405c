"""ctypes binding of include/fabgpu_ecdsa.h (libfabgpu_ecdsa.so).  Fails loudly when the library is absent."""
import ctypes
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
# FABGPU_LIB: development knob, points the binding at another build of the same library (kernel A/B runs)
LIB_PATH = os.environ.get("FABGPU_LIB") or os.path.join(_HERE, "lib", "libfabgpu_ecdsa.so")
SLOTS = 3
CAP_V2_0, CAP_V1_3 = 0, 1      # fabgpu_channel_capability
STATEDB_LEVELDB, STATEDB_COUCHDB = 0, 1             # fabgpu_state_database
STATE_REMOVE = (2 ** 64 - 1, 2 ** 64 - 1)   # fabgpu_state_versions_update: a version that removes the key
UPDATE_WORDS, UPDATE_PUT, UPDATE_DELETE = 14, 1, 2       # fabgpu_block_updates: words per record, its ops
SRC_NONE, SRC_BLOCK, SRC_COMMITTED = 0, 1, 2            # ... and its value and metadata sources
COMMITTED = "committed"                                 # block_updates: a value or metadata the peer reads from its state database
PVT_UPDATE_WORDS, UPDATE_RENEW = 11, 3                  # fabgpu_block_pvt_updates: words per record, the op the peer resolves

OK, E_NO_DEVICE, E_CUDA, E_ARG, E_INJECTED = 0, -1, -2, -3, -4
(ST_VALID, ST_INVALID, ST_ERR_NIL_KEY, ST_ERR_EMPTY_SIG, ST_ERR_EMPTY_DIGEST, ST_ERR_UNMARSHAL, ST_ERR_R_NOT_POSITIVE,
 ST_ERR_S_NOT_POSITIVE, ST_ERR_HIGH_S, ST_ERR_UNSUPPORTED_KEY, ST_ERR_OFF_CURVE) = range(11)

# every symbol include/fabgpu_ecdsa.h declares (tests/test_abi.py checks the header against this and the .so)
EXPORTS = [
    "fabgpu_init", "fabgpu_init_shared", "fabgpu_destroy", "fabgpu_last_error", "fabgpu_device_count", "fabgpu_max_batch",
    "fabgpu_host_buffers", "fabgpu_verify_p256", "fabgpu_verify_p256_async", "fabgpu_wait", "fabgpu_verify_p256_host",
    "fabgpu_verify_p256_device", "fabgpu_bccsp_verify_batch", "fabgpu_bccsp_verify", "fabgpu_gate_signature",
    "fabgpu_test_fieldop", "fabgpu_test_table_entries", "fabgpu_launch_count",
    "fabgpu_keys_register", "fabgpu_key_slot_capacity", "fabgpu_host_key_slots", "fabgpu_verify_p256_keyed",
    "fabgpu_verify_p256_keyed_async", "fabgpu_verify_p256_device_keyed", "fabgpu_last_timing", "fabgpu_build_info",
    "fabgpu_msp_configure", "fabgpu_validate_block", "fabgpu_validate_envelopes", "fabgpu_block_buffer", "fabgpu_block_timing", "fabgpu_sha256_segments",
    "fabgpu_bccsp_verify_batch_async", "fabgpu_bccsp_verify_batch_wait", "fabgpu_bccsp_batch_buffers", "fabgpu_bccsp_verify_batch_inplace_async",
    "fabgpu_msp_identity_groups", "fabgpu_namespace_policies", "fabgpu_msp_principal_bits", "fabgpu_collection_policies",
    "fabgpu_key_policies", "fabgpu_key_policies_update", "fabgpu_channel_capability", "fabgpu_namespace_versions",
    "fabgpu_peer_mask_create", "fabgpu_peer_mask_open", "fabgpu_peer_mask_close", "fabgpu_verify_p256_device_keyed_allgather",
    "fabgpu_validate_block_async", "fabgpu_validate_envelopes_async", "fabgpu_validate_wait", "fabgpu_block_buffer_slot",
    "fabgpu_keys_register_small", "fabgpu_small_slot_capacity", "fabgpu_key_table_stats", "fabgpu_small_table_info",
    "fabgpu_committed_txids", "fabgpu_committed_txids_add", "fabgpu_committed_txids_info", "fabgpu_committed_txids_add_block",
    "fabgpu_state_versions", "fabgpu_state_versions_update", "fabgpu_state_versions_info", "fabgpu_validate_mvcc",
    "fabgpu_state_versions_indexed", "fabgpu_state_index_info", "fabgpu_state_database", "fabgpu_test_couch_values",
    "fabgpu_validate_pvtdata", "fabgpu_msp_identities_add", "fabgpu_block_unknown_identities", "fabgpu_block_updates",
    "fabgpu_block_pvt_updates", "fabgpu_block_update_bytes",
]


class FabGpuError(RuntimeError):
    def __init__(self, code, msg):
        super().__init__("fabgpu error %d: %s" % (code, msg))
        self.code = code


def build(extra=""):
    """Compile the CUDA library in-tree for sm_90a (nvcc cross-compiles without a GPU)."""
    env = dict(os.environ)
    args = ["make", "-s", "-C", os.path.join(_HERE, "csrc")]
    if extra:
        args.append("EXTRA=" + extra)
    subprocess.check_call(args, env=env)


_LIB = None


def lib():
    global _LIB
    if _LIB is None:
        if not os.path.exists(LIB_PATH):
            raise FabGpuError(E_NO_DEVICE, "%s is missing: run __graft_entry__.build() (there is no CPU fallback)" % LIB_PATH)
        L = ctypes.CDLL(LIB_PATH)
        L.fabgpu_last_error.restype = ctypes.c_char_p
        L.fabgpu_last_error.argtypes = [ctypes.c_void_p]
        L.fabgpu_max_batch.restype = ctypes.c_size_t
        L.fabgpu_max_batch.argtypes = [ctypes.c_void_p]
        L.fabgpu_launch_count.restype = ctypes.c_ulonglong
        L.fabgpu_launch_count.argtypes = [ctypes.c_void_p]
        L.fabgpu_init_shared.argtypes = [ctypes.c_void_p, ctypes.c_size_t, ctypes.c_void_p]
        L.fabgpu_destroy.argtypes = [ctypes.c_void_p]
        L.fabgpu_destroy.restype = None
        L.fabgpu_device_count.argtypes = [ctypes.c_void_p]
        _LIB = L
    return _LIB


def _p(a):
    return a.ctypes.data_as(ctypes.c_void_p) if a is not None else None


def _blob(items):
    """byte strings -> (their concatenation, never empty, as uint8; the len(items) + 1 offsets as uint32)"""
    off = np.zeros(len(items) + 1, np.uint32)
    off[1:] = np.cumsum([len(x) for x in items])
    b = np.frombuffer(b"".join(items) or b"\x00", np.uint8)
    return np.ascontiguousarray(b), off


def identity_groups(identities):
    """De-duplication groups for fabgpu_msp_identity_groups: identities = [(serialized SerializedIdentity bytes, mspid, ...)].  Two table
    entries get the same group id when they are the same certificate of the same MSP in byte-different encodings -- the reference's
    policy evaluation de-duplicates signers on Mspid + Id with Id = digest of the certificate's DER (common/policies/policy.go:380-386,
    msp/identities.go:55-76), not on the serialized bytes.  Entries whose PEM does not parse are their own group."""
    import base64
    import hashlib
    import re

    def id_bytes(ser):
        off, out = 0, b""
        while off < len(ser):                                   # SerializedIdentity{mspid = 1, id_bytes = 2}
            key = ser[off]; off += 1
            if key & 7 != 2:
                return None
            ln, shift = 0, 0
            while True:
                c = ser[off]; off += 1
                ln |= (c & 0x7F) << shift
                shift += 7
                if not c & 0x80:
                    break
            if key >> 3 == 2:
                out = ser[off:off + ln]
            off += ln
        return out

    keys, groups = {}, np.zeros(len(identities), np.int32)
    for i, it in enumerate(identities):
        ser, mspid = bytes(it[0]), it[1]
        k = (mspid, ser)
        try:
            m = re.search(rb"-----BEGIN CERTIFICATE-----(.*?)-----END CERTIFICATE-----", id_bytes(ser) or b"", re.S)
            if m:
                k = (mspid, hashlib.sha256(base64.b64decode(b"".join(m.group(1).split()))).digest())
        except Exception:
            pass
        groups[i] = keys.setdefault(k, len(keys))
    return groups


def pack_principal_bits(bits):
    """bool [n_ids, n_principals] -> uint32 [n_ids, ceil(n_principals / 32)], the layout fabgpu_msp_principal_bits reads: bit p % 32
    of word p // 32 of row i is bits[i, p]."""
    b = np.asarray(bits, dtype=bool)
    if b.ndim != 2:
        raise ValueError("principal bits must be a 2-D [n_ids, n_principals] array")
    n_ids, n_pr = b.shape
    W = (n_pr + 31) // 32
    padded = np.zeros((n_ids, 32 * W), np.uint64)
    padded[:, :n_pr] = b
    words = (padded.reshape(n_ids, W, 32) << np.arange(32, dtype=np.uint64)).sum(axis=2)
    return words.astype(np.uint32)


def build_info():
    """(window bits of the G table, window bits of the per-key tables) this library was compiled with."""
    a, b = ctypes.c_int(0), ctypes.c_int(0)
    lib().fabgpu_build_info(ctypes.byref(a), ctypes.byref(b))
    return a.value, b.value


def gate_signature(sig: bytes):
    """fabgpu_gate_signature: host gates only (no GPU).  Returns (status, r32, s32)."""
    r = (ctypes.c_uint8 * 32)()
    s = (ctypes.c_uint8 * 32)()
    buf = (ctypes.c_uint8 * max(1, len(sig))).from_buffer_copy(sig if len(sig) else b"\x00")
    st = lib().fabgpu_gate_signature(buf, ctypes.c_size_t(len(sig)), r, s)
    return st, bytes(r), bytes(s)


class Context:
    """fabgpu_ctx owner.  device_ids=None -> CUDA device 0.  share_tables_with=<Context>: a context on that context's devices that shares
    its point tables and key caches (fabgpu_init_shared; device_ids must then be None), e.g. one per channel of a peer."""

    def __init__(self, max_batch=65536, device_ids=None, share_tables_with=None):
        L = lib()
        self._h = ctypes.c_void_p()
        if share_tables_with is not None:
            if device_ids:
                raise ValueError("a context that shares tables runs on the devices of the context it shares with")
            rc = L.fabgpu_init_shared(share_tables_with._h, ctypes.c_size_t(max_batch), ctypes.byref(self._h))
        elif device_ids:
            arr = (ctypes.c_int * len(device_ids))(*device_ids)
            rc = L.fabgpu_init(arr, ctypes.c_int(len(device_ids)), ctypes.c_size_t(max_batch), ctypes.byref(self._h))
        else:
            rc = L.fabgpu_init(None, ctypes.c_int(0), ctypes.c_size_t(max_batch), ctypes.byref(self._h))
        if rc != OK:
            raise FabGpuError(rc, (L.fabgpu_last_error(None) or b"").decode())
        self.max_batch = max_batch
        self._last_block = {}               # slot -> the bytes its last block was submitted in (block_unknown_identities)

    def close(self):
        if self._h:
            lib().fabgpu_destroy(self._h)
            self._h = ctypes.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _ck(self, rc):
        if rc != OK:
            raise FabGpuError(rc, (lib().fabgpu_last_error(self._h) or b"").decode())

    def last_error(self):
        return (lib().fabgpu_last_error(self._h) or b"").decode()

    def launch_count(self):
        return int(lib().fabgpu_launch_count(self._h))

    def device_count(self):
        return int(lib().fabgpu_device_count(self._h))

    # ---- leaf -------------------------------------------------------------------------------------------
    def host_buffers(self, slot=0):
        """numpy views (no copy) of the slot's pinned SoA buffers: dict qx,qy,e,r,s -> uint8[max_batch,32]; mask, offcurve."""
        ptrs = [ctypes.POINTER(ctypes.c_uint8)() for _ in range(5)]
        mask = ctypes.POINTER(ctypes.c_uint32)()
        off = ctypes.POINTER(ctypes.c_uint32)()
        self._ck(lib().fabgpu_host_buffers(self._h, ctypes.c_int(slot), *[ctypes.byref(p) for p in ptrs], ctypes.byref(mask), ctypes.byref(off)))
        out = {}
        for name, p in zip(("qx", "qy", "e", "r", "s"), ptrs):
            out[name] = np.ctypeslib.as_array(p, shape=(self.max_batch, 32))
        words = (self.max_batch + 31) // 32
        out["mask"] = np.ctypeslib.as_array(mask, shape=(words,))
        out["offcurve"] = np.ctypeslib.as_array(off, shape=(words,))
        return out

    def verify_p256(self, slot, n):
        self._ck(lib().fabgpu_verify_p256(self._h, ctypes.c_int(slot), ctypes.c_size_t(n)))

    def verify_p256_async(self, slot, n):
        self._ck(lib().fabgpu_verify_p256_async(self._h, ctypes.c_int(slot), ctypes.c_size_t(n)))

    def wait(self, slot):
        self._ck(lib().fabgpu_wait(self._h, ctypes.c_int(slot)))

    def verify_p256_host(self, qx, qy, e, r, s):
        """SoA uint8[n,32] arrays in ordinary host memory -> (mask uint32[ceil(n/32)], offcurve uint32[...])."""
        arrs = [np.ascontiguousarray(a, dtype=np.uint8).reshape(-1, 32) for a in (qx, qy, e, r, s)]
        n = arrs[0].shape[0]
        assert all(a.shape[0] == n for a in arrs)
        words = (n + 31) // 32
        mask = np.zeros(max(words, 1), np.uint32)
        off = np.zeros(max(words, 1), np.uint32)
        self._ck(lib().fabgpu_verify_p256_host(self._h, *[_p(a) for a in arrs], ctypes.c_size_t(n), _p(mask), _p(off)))
        return mask[:words], off[:words]

    def verify_p256_device(self, d_qx, d_qy, d_e, d_r, d_s, n, d_mask, d_off=0, stream=0, dev_index=0):
        """Raw device pointers (ints).  Enqueues on `stream` (a cudaStream_t as int) and returns immediately."""
        self._ck(lib().fabgpu_verify_p256_device(self._h, ctypes.c_int(dev_index), ctypes.c_void_p(d_qx), ctypes.c_void_p(d_qy),
                                                 ctypes.c_void_p(d_e), ctypes.c_void_p(d_r), ctypes.c_void_p(d_s), ctypes.c_size_t(n),
                                                 ctypes.c_void_p(d_mask), ctypes.c_void_p(d_off), ctypes.c_void_p(stream)))

    # ---- per-key tables ---------------------------------------------------------------------------------
    def keys_register(self, keys_xy):
        """uint8[K,64] -> int32[K] table slots (-1 = no table)."""
        keys_xy = np.ascontiguousarray(keys_xy, dtype=np.uint8).reshape(-1, 64)
        slots = np.full(keys_xy.shape[0], -1, np.int32)
        self._ck(lib().fabgpu_keys_register(self._h, _p(keys_xy), ctypes.c_int(keys_xy.shape[0]), _p(slots)))
        return slots

    def key_slot_capacity(self):
        return int(lib().fabgpu_key_slot_capacity(self._h))

    def keys_register_small(self, keys_xy):
        """uint8[K,64] -> int32[K] small-table handles (<= -2; -1 = no slot could be had)."""
        keys_xy = np.ascontiguousarray(keys_xy, dtype=np.uint8).reshape(-1, 64)
        handles = np.full(keys_xy.shape[0], -1, np.int32)
        self._ck(lib().fabgpu_keys_register_small(self._h, _p(keys_xy), ctypes.c_int(keys_xy.shape[0]), _p(handles)))
        return handles

    @staticmethod
    def small_raw_codes(handles):
        """small handles -> the raw device codes fabgpu_verify_p256_device_keyed takes (-2 - slot)."""
        h = np.asarray(handles, np.int64)
        return np.where(h <= -2, -2 - ((-2 - h) & 0xFFFFF), -1).astype(np.int32)

    def key_table_stats(self):
        """{'big': window tables alive, 'small': small tables alive, 'small_built': ..., 'small_recycled': ...}"""
        out = (ctypes.c_ulonglong * 4)()
        self._ck(lib().fabgpu_key_table_stats(self._h, out))
        return {"big": int(out[0]), "small": int(out[1]), "small_built": int(out[2]), "small_recycled": int(out[3])}

    @staticmethod
    def small_table_info():
        """(signed window bits, windows, bytes per table) of the small key tables."""
        wb, nw, nb = ctypes.c_int(0), ctypes.c_int(0), ctypes.c_size_t(0)
        lib().fabgpu_small_table_info(ctypes.byref(wb), ctypes.byref(nw), ctypes.byref(nb))
        return wb.value, nw.value, nb.value

    def small_slot_capacity(self):
        return int(lib().fabgpu_small_slot_capacity(self._h))

    def host_key_slots(self, slot=0):
        p = ctypes.POINTER(ctypes.c_int32)()
        self._ck(lib().fabgpu_host_key_slots(self._h, ctypes.c_int(slot), ctypes.byref(p)))
        return np.ctypeslib.as_array(p, shape=(self.max_batch,))

    def verify_p256_keyed(self, slot, n):
        self._ck(lib().fabgpu_verify_p256_keyed(self._h, ctypes.c_int(slot), ctypes.c_size_t(n)))

    def verify_p256_keyed_async(self, slot, n):
        self._ck(lib().fabgpu_verify_p256_keyed_async(self._h, ctypes.c_int(slot), ctypes.c_size_t(n)))

    def verify_p256_device_keyed(self, all_cached, d_key_slot, d_qx, d_qy, d_e, d_r, d_s, n, d_mask, d_off=0, stream=0, dev_index=0):
        self._ck(lib().fabgpu_verify_p256_device_keyed(self._h, ctypes.c_int(dev_index), ctypes.c_int(int(all_cached)),
                                                       ctypes.c_void_p(d_key_slot), ctypes.c_void_p(d_qx), ctypes.c_void_p(d_qy),
                                                       ctypes.c_void_p(d_e), ctypes.c_void_p(d_r), ctypes.c_void_p(d_s), ctypes.c_size_t(n),
                                                       ctypes.c_void_p(d_mask), ctypes.c_void_p(d_off), ctypes.c_void_p(stream)))

    # ---- bitmask exchange over peer memory (one process per GPU) ------------------------------------------
    def peer_mask_create(self, world, rank, words_per_rank, dev_index=0):
        h = np.zeros(64, np.uint8)
        self._ck(lib().fabgpu_peer_mask_create(self._h, ctypes.c_int(dev_index), ctypes.c_int(world), ctypes.c_int(rank), ctypes.c_size_t(words_per_rank), _p(h)))
        return h

    def peer_mask_open(self, handles, dev_index=0):
        handles = np.ascontiguousarray(handles, dtype=np.uint8).reshape(-1)
        self._ck(lib().fabgpu_peer_mask_open(self._h, ctypes.c_int(dev_index), _p(handles)))

    def peer_mask_close(self, dev_index=0):
        self._ck(lib().fabgpu_peer_mask_close(self._h, ctypes.c_int(dev_index)))

    def verify_p256_device_keyed_allgather(self, all_cached, d_key_slot, d_qx, d_qy, d_e, d_r, d_s, n, step, stream=0, dev_index=0):
        """Returns the device pointer (int) of the assembled world x words_per_rank mask words of this step."""
        out = ctypes.c_void_p(0)
        self._ck(lib().fabgpu_verify_p256_device_keyed_allgather(self._h, ctypes.c_int(dev_index), ctypes.c_int(1 if all_cached else 0), ctypes.c_void_p(d_key_slot),
                                                                 ctypes.c_void_p(d_qx), ctypes.c_void_p(d_qy), ctypes.c_void_p(d_e), ctypes.c_void_p(d_r),
                                                                 ctypes.c_void_p(d_s), ctypes.c_size_t(n), ctypes.c_uint32(step), ctypes.byref(out), ctypes.c_void_p(stream)))
        return int(out.value or 0)

    # ---- bccsp level ------------------------------------------------------------------------------------
    @staticmethod
    def _batch_args(keys_xy, key_idx, digests, dig_off, sigs, sig_off):
        keys_xy = np.ascontiguousarray(keys_xy, dtype=np.uint8).reshape(-1, 64)
        key_idx = np.ascontiguousarray(key_idx, dtype=np.int32)
        digests = np.ascontiguousarray(digests, dtype=np.uint8).reshape(-1)
        sigs = np.ascontiguousarray(sigs, dtype=np.uint8).reshape(-1)
        dig_off = np.ascontiguousarray(dig_off, dtype=np.uint32)
        sig_off = np.ascontiguousarray(sig_off, dtype=np.uint32)
        if digests.size == 0:
            digests = np.zeros(1, np.uint8)
        if sigs.size == 0:
            sigs = np.zeros(1, np.uint8)
        return keys_xy, key_idx, digests, dig_off, sigs, sig_off

    def bccsp_verify_batch(self, keys_xy, key_idx, digests, dig_off, sigs, sig_off):
        keys_xy, key_idx, digests, dig_off, sigs, sig_off = self._batch_args(keys_xy, key_idx, digests, dig_off, sigs, sig_off)
        n = key_idx.shape[0]
        status = np.full(max(n, 1), 255, np.uint8)
        self._ck(lib().fabgpu_bccsp_verify_batch(self._h, _p(keys_xy), ctypes.c_int(keys_xy.shape[0]), _p(key_idx), _p(digests), _p(dig_off),
                                                 _p(sigs), _p(sig_off), ctypes.c_size_t(n), _p(status)))
        return status[:n]

    def bccsp_verify_batch_async(self, slot, keys_xy, key_idx, digests, dig_off, sigs, sig_off):
        """First half of bccsp_verify_batch on one of the FABGPU_SLOTS slots; returns n for the matching _wait."""
        keys_xy, key_idx, digests, dig_off, sigs, sig_off = self._batch_args(keys_xy, key_idx, digests, dig_off, sigs, sig_off)
        n = key_idx.shape[0]
        self._ck(lib().fabgpu_bccsp_verify_batch_async(self._h, ctypes.c_int(slot), _p(keys_xy), ctypes.c_int(keys_xy.shape[0]), _p(key_idx),
                                                       _p(digests), _p(dig_off), _p(sigs), _p(sig_off), ctypes.c_size_t(n)))
        return n

    def bccsp_verify_batch_wait(self, slot, n, out=None):
        status = out if out is not None else np.full(max(n, 1), 255, np.uint8)
        self._ck(lib().fabgpu_bccsp_verify_batch_wait(self._h, ctypes.c_int(slot), _p(status), ctypes.c_size_t(n)))
        return status[:n]

    def bccsp_batch_buffers(self, slot, n_cap, sig_bytes_cap, dig_bytes_cap, k_cap):
        """numpy views (no copy) of the slot's pinned batch buffers: dict keys_xy uint8[k_cap,64], key_idx int32[n_cap], digests uint8[dig_bytes_cap],
        dig_off uint32[n_cap+1], sigs uint8[sig_bytes_cap], sig_off uint32[n_cap+1].  Fill them, then bccsp_verify_batch_inplace_async."""
        pk, pd, ps = (ctypes.POINTER(ctypes.c_uint8)() for _ in range(3))
        pi = ctypes.POINTER(ctypes.c_int32)()
        pdo, pso = ctypes.POINTER(ctypes.c_uint32)(), ctypes.POINTER(ctypes.c_uint32)()
        self._ck(lib().fabgpu_bccsp_batch_buffers(self._h, ctypes.c_int(slot), ctypes.c_size_t(n_cap), ctypes.c_size_t(sig_bytes_cap), ctypes.c_size_t(dig_bytes_cap),
                                                  ctypes.c_int(k_cap), ctypes.byref(pk), ctypes.byref(pi), ctypes.byref(pd), ctypes.byref(pdo), ctypes.byref(ps), ctypes.byref(pso)))
        A = np.ctypeslib.as_array
        return {"keys_xy": A(pk, shape=(max(k_cap, 1), 64)), "key_idx": A(pi, shape=(max(n_cap, 1),)), "digests": A(pd, shape=(max(dig_bytes_cap, 1),)),
                "dig_off": A(pdo, shape=(n_cap + 1,)), "sigs": A(ps, shape=(max(sig_bytes_cap, 1),)), "sig_off": A(pso, shape=(n_cap + 1,))}

    def bccsp_fill_batch_buffers(self, slot, keys_xy, key_idx, digests, dig_off, sigs, sig_off):
        """Convenience: reserve + copy a batch into the slot's pinned buffers once; returns (K, n) for bccsp_verify_batch_inplace_async."""
        keys_xy, key_idx, digests, dig_off, sigs, sig_off = self._batch_args(keys_xy, key_idx, digests, dig_off, sigs, sig_off)
        n, K = key_idx.shape[0], keys_xy.shape[0]
        hb = self.bccsp_batch_buffers(slot, n, int(sig_off[n]), int(dig_off[n]), K)
        hb["keys_xy"][:K] = keys_xy; hb["key_idx"][:n] = key_idx
        hb["digests"][: int(dig_off[n])] = digests[: int(dig_off[n])]; hb["dig_off"][: n + 1] = dig_off
        hb["sigs"][: int(sig_off[n])] = sigs[: int(sig_off[n])]; hb["sig_off"][: n + 1] = sig_off
        return K, n

    def bccsp_verify_batch_inplace_async(self, slot, K, n):
        self._ck(lib().fabgpu_bccsp_verify_batch_inplace_async(self._h, ctypes.c_int(slot), ctypes.c_int(K), ctypes.c_size_t(n)))
        return n

    def bccsp_verify(self, key_xy, sig, digest):
        """One sw.CSP.Verify call -> (valid: bool, err: str|None) with the reference's error strings."""
        valid = ctypes.c_int(0)
        err = ctypes.create_string_buffer(1024)
        kb = (ctypes.c_uint8 * 64).from_buffer_copy(key_xy) if key_xy is not None else None
        sb = (ctypes.c_uint8 * max(1, len(sig or b""))).from_buffer_copy(sig if sig else b"\x00")
        db = (ctypes.c_uint8 * max(1, len(digest or b""))).from_buffer_copy(digest if digest else b"\x00")
        self._ck(lib().fabgpu_bccsp_verify(self._h, kb, sb, ctypes.c_size_t(len(sig or b"")), db, ctypes.c_size_t(len(digest or b"")),
                                           ctypes.byref(valid), err, ctypes.c_size_t(1024)))
        e = err.value.decode()
        return bool(valid.value), (e if e else None)

    # ---- block level ------------------------------------------------------------------------------------
    def msp_configure(self, identities, policy_nodes, principals, channel, policies=None):
        """identities: list of (serialized: bytes, mspid: str, key_xy: 64 bytes, valid: bool).  policy_nodes may hold several policy
        trees; policies = {namespace: root node index} names the tree of each chaincode namespace (None: node 0 for every namespace).
        The identities' de-duplication groups (Mspid + certificate, identity_groups) are installed as well."""
        idb, ido = _blob([bytes(i[0]) for i in identities])
        mb, mo = _blob([i[1].encode() for i in identities])
        keys = np.ascontiguousarray(np.frombuffer(b"".join(bytes(i[2]) for i in identities) or b"\x00" * 64, np.uint8))
        valid = np.array([1 if i[3] else 0 for i in identities] or [0], np.uint8)
        nodes = np.ascontiguousarray(policy_nodes, dtype=np.int32).reshape(-1, 4)
        pbb, pbo = _blob([p.encode() for p in principals])
        self._ck(lib().fabgpu_msp_configure(self._h, _p(idb), _p(ido), _p(mb), _p(mo), _p(keys), _p(valid), ctypes.c_int(len(identities)),
                                            _p(nodes), ctypes.c_int(nodes.shape[0]), _p(pbb), _p(pbo), ctypes.c_int(len(principals)),
                                            ctypes.c_char_p(channel.encode())))
        if identities:
            groups = np.ascontiguousarray(identity_groups(identities), np.int32)
            self._ck(lib().fabgpu_msp_identity_groups(self._h, _p(groups), ctypes.c_int(len(identities))))
        names = sorted(policies) if policies else []
        nb, no = _blob([n.encode() for n in names])
        roots = np.array([policies[n] for n in names] or [0], np.int32)
        self._ck(lib().fabgpu_namespace_policies(self._h, _p(nb), _p(no), _p(roots), ctypes.c_int(len(names))))
        self._ns_names = names
        self._n_principals = len(principals)

    def channel_capability(self, cap):
        """cap: CAP_V2_0 (the default after msp_configure) for a channel with V2_0Validation, CAP_V1_3 for a V1_3 / V1_4_2 / V1_4_3
        channel: the v1.4 validator with the builtin v13 VSCC (fabgpu_channel_capability)."""
        self._ck(lib().fabgpu_channel_capability(self._h, ctypes.c_int(cap)))

    def namespace_versions(self, versions):
        """versions: {namespace: lscc ChaincodeData.Version} for the namespaces msp_configure's policies named; a namespace left out has
        no version (its invocations are 254 in CAP_V1_3 mode), so None or an empty dict clears them (fabgpu_namespace_versions)."""
        names = getattr(self, "_ns_names", [])
        vb, vo = _blob([(versions or {}).get(n, "").encode() for n in names])
        self._ck(lib().fabgpu_namespace_versions(self._h, _p(vb), _p(vo), ctypes.c_int(len(names))))

    def msp_principal_bits(self, bits):
        """bits: bool [n_ids, n_principals], bits[i, p] = identity i satisfies principal p (msp Identity.SatisfiesPrincipal), for the
        identities and principals of the last msp_configure, in that order.  SignedBy(p) then matches by these bits instead of by
        MSP id.  None, or no rows, removes them."""
        b = np.zeros((0, 0), bool) if bits is None else np.asarray(bits, dtype=bool)
        words = np.ascontiguousarray(pack_principal_bits(b)).reshape(-1)
        words = words if words.size else np.zeros(1, np.uint32)
        self._ck(lib().fabgpu_msp_principal_bits(self._h, _p(words), ctypes.c_int(b.shape[0]), ctypes.c_int(b.shape[1])))

    def msp_identities_add(self, identities, groups=None, bits=None):
        """Admits identities into the table msp_configure installed, without draining the blocks in flight (fabgpu_msp_identities_add):
        seen by every block submitted after this returns, by none submitted before.  identities: list of (serialized, mspid, key_xy,
        valid) as for msp_configure.  groups: one de-duplication id each, required iff a group table is installed (msp_configure
        installs one; identity_groups over the whole table gives consistent ids); bits: bool [n, n_principals], required iff
        principal bits are installed."""
        idb, ido = _blob([bytes(i[0]) for i in identities])
        mb, mo = _blob([i[1].encode() for i in identities])
        keys = np.ascontiguousarray(np.frombuffer(b"".join(bytes(i[2]) for i in identities) or b"\x00" * 64, np.uint8))
        valid = np.array([1 if i[3] else 0 for i in identities] or [0], np.uint8)
        g = None if groups is None else np.ascontiguousarray(np.asarray(list(groups) or [0], np.int32))
        if g is not None and identities and g.shape[0] != len(identities):
            raise ValueError("one group per identity")
        w = None
        if bits is not None:
            # the library reads one row of the configured principals' width per identity
            b = np.asarray(bits, dtype=bool)
            n_pr = getattr(self, "_n_principals", 0)
            if b.size == 0 and not identities:
                b = np.zeros((0, n_pr), bool)
            if b.ndim != 2 or b.shape != (len(identities), n_pr):
                raise ValueError("bits must be a [n_identities, n_principals] array over msp_configure's %d principals" % n_pr)
            w = np.ascontiguousarray(pack_principal_bits(b)).reshape(-1)
            w = w if w.size else np.zeros(1, np.uint32)
        self._ck(lib().fabgpu_msp_identities_add(self._h, _p(idb), _p(ido), _p(mb), _p(mo), _p(keys), _p(valid), _p(g), _p(w),
                                                 ctypes.c_int(len(identities))))

    def block_unknown_identities(self, slot):
        """The identities the finished block on `slot` looked up and did not find (fabgpu_block_unknown_identities), distinct, in order
        of first appearance: [(serialized bytes, first tx)].  Call it between validate_wait(slot) and the slot's next submit; the
        block's bytes must still be alive (they are read back from the buffer the block was submitted in)."""
        n, cap = ctypes.c_size_t(0), 1024
        while True:
            out = np.zeros(3 * cap, np.uint32)
            self._ck(lib().fabgpu_block_unknown_identities(self._h, ctypes.c_int(slot), _p(out), ctypes.c_size_t(cap), ctypes.byref(n)))
            if n.value <= cap:
                break
            cap = n.value
        src = self._last_block.get(slot)
        if src is None:
            raise FabGpuError(E_ARG, "no block submitted on this slot through this binding")
        return [(bytes(src[int(out[3 * i]): int(out[3 * i]) + int(out[3 * i + 1])]), int(out[3 * i + 2])) for i in range(n.value)]

    def block_updates(self, slot, block_num):
        """The update batch of the block validate_mvcc(slot, block_num) last ran on (fabgpu_block_updates): [(tx, op, ns, coll, key, value,
        metadata)] in the library's order -- op "put" or "del"; ns, coll (b"" for a public key) and key as bytes; value the bytes (read back
        from the buffer the block was submitted in), COMMITTED (the peer's GetState supplies it) or None for a delete; metadata the
        Serialize bytes, None (nil) or COMMITTED.  None when the batch is incomplete and the peer builds it itself."""
        n = (ctypes.c_size_t * 2)()
        complete = ctypes.c_int(0)
        rec_cap, meta_cap = 1024, 1 << 16
        while True:
            rec = np.zeros(UPDATE_WORDS * rec_cap, np.uint32)
            meta = np.zeros(meta_cap, np.uint8)
            self._ck(lib().fabgpu_block_updates(self._h, ctypes.c_int(slot), ctypes.c_uint64(block_num), _p(rec), ctypes.c_size_t(rec_cap), _p(meta),
                                                ctypes.c_size_t(meta_cap), n, ctypes.byref(complete)))
            if n[0] <= rec_cap and n[1] <= meta_cap:
                break
            rec_cap, meta_cap = max(rec_cap, n[0]), max(meta_cap, n[1])
        if not complete.value:
            return None
        src = memoryview(self._last_block[slot]).cast("B")
        meta = meta.tobytes()
        out = []
        for w in rec[: UPDATE_WORDS * n[0]].reshape(-1, UPDATE_WORDS).tolist():
            value = None if w[2] == SRC_NONE else bytes(src[w[10]:w[10] + w[11]]) if w[2] == SRC_BLOCK else COMMITTED
            md = None if w[3] == SRC_NONE else meta[w[12]:w[12] + w[13]] if w[3] == SRC_BLOCK else COMMITTED
            out.append((w[0], "put" if w[1] == UPDATE_PUT else "del", bytes(src[w[4]:w[4] + w[5]]), bytes(src[w[6]:w[6] + w[7]]),
                        bytes(src[w[8]:w[8] + w[9]]), value, md))
        return out

    def block_update_bytes(self, slot, block_num, committed=()):
        """The bytes deterministicBytesForPubAndHashUpdates returns for the update batch of the block validate_mvcc(slot, block_num) last
        ran on (fabgpu_block_update_bytes): the input of the block's commit hash.  committed: the values of block_updates' COMMITTED-value
        records, in record order (GetState / GetValueHash).  bytes, or None when incomplete and the peer builds them itself."""
        committed = [bytes(v) for v in committed]
        blob, off = _blob(committed)
        n = ctypes.c_size_t(0)
        complete = ctypes.c_int(0)
        cap = 1 << 16
        while True:
            out = np.zeros(cap, np.uint8)
            self._ck(lib().fabgpu_block_update_bytes(self._h, ctypes.c_int(slot), ctypes.c_uint64(block_num), _p(blob), _p(off),
                                                     ctypes.c_size_t(len(committed)), _p(out), ctypes.c_size_t(cap), ctypes.byref(n),
                                                     ctypes.byref(complete)))
            if n.value <= cap:
                break
            cap = n.value
        return out[: n.value].tobytes() if complete.value else None

    def block_pvt_updates(self, slot, block_num, pvt):
        """The private update batch of the block validate_mvcc(slot, block_num) last ran on (fabgpu_block_pvt_updates); pvt maps SeqInBlock
        -> marshalled rwset.TxPvtReadWriteSet, as validate_pvtdata takes it.  Returns (verdict, status, records): verdict and status as
        validate_pvtdata gives them with the stage's flags; records None when the batch is incomplete (the peer builds it itself), else
        [(tx, op, ns, coll, key, value, hashed_index)] in the library's order -- op "put", "del" or "renew"; ns, coll, key and value (a put's;
        None otherwise) as bytes; hashed_index the index of the hashed PUT record in block_updates' list for a "renew", else None."""
        seqs = sorted(pvt)
        items = [bytes(pvt[k]) for k in seqs]
        blob, off = _blob(items)
        sq = np.array(seqs or [0], np.uint32)
        st = np.zeros(3 * max(len(seqs), 1), np.int32)
        out = np.zeros(4, np.int32)
        n = ctypes.c_size_t(0)
        complete = ctypes.c_int(0)
        cap = 1024
        while True:
            rec = np.zeros(PVT_UPDATE_WORDS * cap, np.uint32)
            self._ck(lib().fabgpu_block_pvt_updates(self._h, ctypes.c_int(slot), ctypes.c_uint64(block_num), _p(blob), _p(off), _p(sq),
                                                    ctypes.c_size_t(len(seqs)), _p(st), _p(out), _p(rec), ctypes.c_size_t(cap), ctypes.byref(n),
                                                    ctypes.byref(complete)))
            if n.value <= cap:
                break
            cap = n.value
        verdict = tuple(int(x) for x in out)
        status = {k: tuple(int(x) for x in st[3 * i:3 * i + 3]) for i, k in enumerate(seqs)}
        if not complete.value:
            return verdict, status, None
        src = bytes(blob)
        ops = {UPDATE_PUT: "put", UPDATE_DELETE: "del", UPDATE_RENEW: "renew"}
        records = []
        for w in rec[: PVT_UPDATE_WORDS * n.value].reshape(-1, PVT_UPDATE_WORDS).tolist():
            records.append((w[0], ops[w[1]], src[w[2]:w[2] + w[3]], src[w[4]:w[4] + w[5]], src[w[6]:w[6] + w[7]],
                            src[w[8]:w[8] + w[9]] if w[1] == UPDATE_PUT else None, w[10] if w[1] == UPDATE_RENEW else None))
        return verdict, status, records

    def collection_policies(self, table):
        """table: {(namespace, collection): root node index} -- the endorsement policy a write to that private-data collection is checked
        against instead of the chaincode's (fabgpu_collection_policies).  None or an empty dict removes the table."""
        keys = sorted(table) if table else []
        nb, no = _blob([ns.encode() for ns, _ in keys])
        cb, co = _blob([c.encode() for _, c in keys])
        roots = np.array([table[k] for k in keys] or [0], np.int32)
        self._ck(lib().fabgpu_collection_policies(self._h, _p(nb), _p(no), _p(cb), _p(co), _p(roots), ctypes.c_int(len(keys))))

    def key_policies(self, nodes, table):
        """nodes: (n, 4) int32 policy nodes of the validation parameters (NOutOf / SignedBy, child indices within `nodes`, SignedBy indexing
        msp_configure's principals); table: {(namespace, collection, key): root} -- the root node of that key's validation parameter, or -2
        when the device may not decide it.  collection is "" for a public key; key is str or bytes (the 32-byte key hash for a collection
        key).  Replaces the key policy table (fabgpu_key_policies); no nodes and an empty table remove it."""
        self._key_policies(lib().fabgpu_key_policies, nodes, table)

    def key_policies_update(self, nodes, table):
        """Upserts into the installed key policy table (fabgpu_key_policies_update): same arguments, root -1 removes the key."""
        self._key_policies(lib().fabgpu_key_policies_update, nodes, table)

    def _key_policies(self, fn, nodes, table):
        b = lambda x: x.encode() if isinstance(x, str) else bytes(x)
        keys = list(table) if table else []
        nb, no = _blob([b(k[0]) for k in keys])
        cb, co = _blob([b(k[1]) for k in keys])
        kb, ko = _blob([b(k[2]) for k in keys])
        roots = np.array([table[k] for k in keys] or [0], np.int32)
        nd = np.ascontiguousarray(np.asarray(nodes if nodes is not None and len(nodes) else np.zeros((0, 4)), dtype=np.int32).reshape(-1, 4))
        ndp = nd if nd.shape[0] else np.zeros((1, 4), np.int32)
        self._ck(fn(self._h, _p(ndp), ctypes.c_int(nd.shape[0]), _p(nb), _p(no), _p(cb), _p(co), _p(kb), _p(ko), _p(roots), ctypes.c_int(len(keys))))

    def committed_txids(self, ids, kinds=None, capacity=0):
        """Replaces the ledger's committed tx-id set (fabgpu_committed_txids).  ids: tx id strings (str or bytes, as in ChannelHeader.tx_id);
        kinds: one per id, 0 = committed (a transaction with that id is DUPLICATE_TXID), 1 = indexed but GetTransactionByID fails (254);
        None = all 0.  capacity sizes the table for that many ids.  No ids and capacity 0 remove the set."""
        self._committed_txids(lib().fabgpu_committed_txids, ids, kinds, (ctypes.c_size_t(capacity),))

    def committed_txids_add(self, ids, kinds=None):
        """Upserts ids into the installed set (fabgpu_committed_txids_add) without draining the blocks in flight: seen by every block
        submitted after this returns, by none submitted before."""
        self._committed_txids(lib().fabgpu_committed_txids_add, ids, kinds, ())

    def committed_txids_add_block(self, slot):
        """Upserts the ids the block store indexes for the block submitted on `slot` (fabgpu_committed_txids_add_block), extracted on the
        device: call it after validate_*_async(slot) (or a blocking validate_* call, slot 0) and before the slot's next submit."""
        self._ck(lib().fabgpu_committed_txids_add_block(self._h, ctypes.c_int(slot)))

    def committed_txids_info(self):
        """(distinct ids held, table slots)"""
        out = (ctypes.c_ulonglong * 2)()
        self._ck(lib().fabgpu_committed_txids_info(self._h, out))
        return int(out[0]), int(out[1])

    def _committed_txids(self, fn, ids, kinds, extra):
        ids = [x.encode() if isinstance(x, str) else bytes(x) for x in ids]
        b, o = _blob(ids)
        k = None if kinds is None else np.ascontiguousarray(np.asarray(list(kinds) or [0], np.uint8))
        if k is not None and len(ids) and k.shape[0] != len(ids):
            raise ValueError("one kind per id")
        self._ck(fn(self._h, _p(b), _p(o), _p(k), ctypes.c_size_t(len(ids)), *extra))

    def state_versions(self, entries, height, capacity=0):
        """Replaces the world-state version table of the MVCC stage (fabgpu_state_versions).  entries: [((namespace, collection, key),
        (block_num, tx_num))] -- collection "" for a public key, key str or bytes (the 32-byte key hash for a collection key); height:
        committed blocks, the next block validate_mvcc checks.  capacity sizes the table for that many keys.  No entries and capacity 0
        remove the table."""
        self._state_versions(lib().fabgpu_state_versions, entries, height, (ctypes.c_size_t(capacity),))

    def state_versions_indexed(self, entries, height, capacity=0):
        """state_versions, and an ordered index of the public keys (fabgpu_state_versions_indexed): while it is installed validate_mvcc
        decides range queries (phantom reads) instead of giving them 254.  state_versions drops the index."""
        self._state_versions(lib().fabgpu_state_versions_indexed, entries, height, (ctypes.c_size_t(capacity),))

    def state_index_info(self):
        """(index entries the table holds, entries including dead ones, index bytes on the device); zeros without an index"""
        out = (ctypes.c_ulonglong * 3)()
        self._ck(lib().fabgpu_state_index_info(self._h, out))
        return tuple(int(x) for x in out)

    def state_database(self, kind):
        """The state database validate_mvcc restates (fabgpu_state_database): STATEDB_LEVELDB (the default) or STATEDB_COUCHDB, which
        adds CouchDB's key and value checks (INVALID_WRITESET, 24) and makes the install calls refuse public keys CouchDB cannot hold."""
        self._ck(lib().fabgpu_state_database(self._h, ctypes.c_int(kind)))

    def test_couch_values(self, values, path=0):
        """The device's verdict bits of CouchDB's value check on each of the byte strings (fabgpu_test_couch_values): path 0 chooses
        the scan by length as validate_mvcc does, 1 forces the one-thread scan, 2 the CTA scan"""
        b, o = _blob([bytes(v) for v in values])
        out = np.zeros(max(len(values), 1), np.uint32)
        self._ck(lib().fabgpu_test_couch_values(self._h, _p(b), _p(o), ctypes.c_size_t(len(values)), ctypes.c_int(path), _p(out)))
        return out[: len(values)]

    def state_versions_update(self, entries, height):
        """Upserts entries (fabgpu_state_versions_update); a version of STATE_REMOVE removes the key.  A height above the table's
        closes a block validate_mvcc left open."""
        self._state_versions(lib().fabgpu_state_versions_update, entries, height, ())

    def state_versions_info(self):
        """(keys held, table slots, height, keys unknown)"""
        out = (ctypes.c_ulonglong * 4)()
        self._ck(lib().fabgpu_state_versions_info(self._h, out))
        return tuple(int(x) for x in out)

    def validate_mvcc(self, slot, block_num, tv_flags):
        """The MVCC stage of the block validate_wait(slot) returned (fabgpu_validate_mvcc): tv_flags are the validator's flags, the result
        the committed ones (VALID, 11 or 254 for each VALID, the others copied).  Applies the block to the table at height block_num."""
        tv = np.ascontiguousarray(np.asarray(tv_flags, np.uint8))
        flags = np.zeros(max(tv.shape[0], 1), np.uint8)
        self._ck(lib().fabgpu_validate_mvcc(self._h, ctypes.c_int(slot), ctypes.c_uint64(block_num), _p(tv if tv.size else flags), _p(flags),
                                            ctypes.c_size_t(tv.shape[0])))
        return flags[: tv.shape[0]]

    def validate_pvtdata(self, slot, flags, pvt):
        """The private-data check of the block validate_wait(slot) returned (fabgpu_validate_pvtdata): flags are the block's final flags,
        pvt maps SeqInBlock -> marshalled rwset.TxPvtReadWriteSet.  Returns (verdict, status): verdict = (code, seq, ns, coll) with code 0
        OK, 1 mismatch, 254; status[seq] = (code, ns, coll) per entry, code 0 OK, 1 mismatch, 2 skipped, 254."""
        fl = np.ascontiguousarray(np.asarray(flags, np.uint8))
        seqs = sorted(pvt)
        blob, off = _blob([bytes(pvt[k]) for k in seqs])
        sq = np.array(seqs or [0], np.uint32)
        st = np.zeros(3 * max(len(seqs), 1), np.int32)
        out = np.zeros(4, np.int32)
        self._ck(lib().fabgpu_validate_pvtdata(self._h, ctypes.c_int(slot), _p(fl if fl.size else out), ctypes.c_size_t(fl.shape[0]), _p(blob), _p(off),
                                               _p(sq), ctypes.c_size_t(len(seqs)), _p(st), _p(out)))
        return tuple(int(x) for x in out), {k: tuple(int(x) for x in st[3 * i:3 * i + 3]) for i, k in enumerate(seqs)}

    def _state_versions(self, fn, entries, height, extra):
        b = lambda x: x.encode() if isinstance(x, str) else bytes(x)
        entries = list(entries)
        nb, no = _blob([b(k[0]) for k, _ in entries])
        cb, co = _blob([b(k[1]) for k, _ in entries])
        kb, ko = _blob([b(k[2]) for k, _ in entries])
        ver = np.ascontiguousarray(np.array([x for _, v in entries for x in v] or [0], np.uint64))
        self._ck(fn(self._h, _p(nb), _p(no), _p(cb), _p(co), _p(kb), _p(ko), _p(ver), ctypes.c_size_t(len(entries)), ctypes.c_uint64(height), *extra))

    def block_buffer(self, nbytes, slot=0):
        """Pinned staging buffer (numpy view) for block bytes; one per slot."""
        p = ctypes.POINTER(ctypes.c_uint8)()
        self._ck(lib().fabgpu_block_buffer_slot(self._h, ctypes.c_int(slot), ctypes.c_size_t(nbytes), ctypes.byref(p)))
        return np.ctypeslib.as_array(p, shape=(nbytes,))

    def validate_envelopes_async(self, slot, blob, env_off):
        """First half of validate_envelopes on one of the FABGPU_SLOTS slots.  `blob` must stay alive and unchanged until
        validate_wait(slot) returns (it is kept referenced here).  Returns the number of envelopes."""
        arr = np.frombuffer(blob, np.uint8) if isinstance(blob, (bytes, bytearray)) else blob
        env_off = np.ascontiguousarray(env_off, dtype=np.uint32)
        n_env = env_off.shape[0] - 1
        self._inflight = getattr(self, "_inflight", {})
        self._inflight[slot] = (arr, env_off)
        self._last_block[slot] = arr
        self._ck(lib().fabgpu_validate_envelopes_async(self._h, ctypes.c_int(slot), _p(arr), _p(env_off), ctypes.c_size_t(n_env)))
        return n_env

    def validate_block_async(self, slot, block):
        arr = np.frombuffer(block, np.uint8) if isinstance(block, (bytes, bytearray)) else block
        self._inflight = getattr(self, "_inflight", {})
        self._inflight[slot] = (arr,)
        self._last_block[slot] = arr
        self._ck(lib().fabgpu_validate_block_async(self._h, ctypes.c_int(slot), _p(arr), ctypes.c_size_t(arr.shape[0])))
        return max(16, arr.shape[0] // 2)

    def validate_wait(self, slot, max_tx):
        flags = np.full(max(max_tx, 1), 254, np.uint8)
        n = ctypes.c_size_t(0)
        try:
            self._ck(lib().fabgpu_validate_wait(self._h, ctypes.c_int(slot), _p(flags), ctypes.c_size_t(flags.shape[0]), ctypes.byref(n)))
        finally:
            getattr(self, "_inflight", {}).pop(slot, None)
        return flags[: n.value]

    def validate_block(self, block, max_tx=None):
        """block: bytes or a uint8 numpy array (e.g. a slice of block_buffer()).  Returns the TRANSACTIONS_FILTER bytes."""
        arr = np.frombuffer(block, np.uint8) if isinstance(block, (bytes, bytearray)) else block
        self._last_block[0] = arr
        cap = max_tx or max(16, arr.shape[0] // 64)
        flags = np.full(cap, 254, np.uint8)
        n = ctypes.c_size_t(0)
        self._ck(lib().fabgpu_validate_block(self._h, _p(arr), ctypes.c_size_t(arr.shape[0]), _p(flags), ctypes.c_size_t(cap), ctypes.byref(n)))
        return flags[: n.value]

    def validate_envelopes(self, blob, env_off):
        """blob: uint8 array holding the envelopes back to back; env_off: uint32[n+1].  Returns the flags."""
        arr = np.frombuffer(blob, np.uint8) if isinstance(blob, (bytes, bytearray)) else blob
        env_off = np.ascontiguousarray(env_off, dtype=np.uint32)
        n_env = env_off.shape[0] - 1
        self._last_block[0] = arr
        flags = np.full(max(n_env, 1), 254, np.uint8)
        n = ctypes.c_size_t(0)
        self._ck(lib().fabgpu_validate_envelopes(self._h, _p(arr), _p(env_off), ctypes.c_size_t(n_env), _p(flags), ctypes.c_size_t(max(n_env, 1)),
                                                 ctypes.byref(n)))
        return flags[: n.value]

    def block_timing(self):
        out = (ctypes.c_double * 10)()
        self._ck(lib().fabgpu_block_timing(self._h, out))
        return [float(x) for x in out]

    def sha256_segments(self, buf, jobs):
        """jobs: uint32[n,6] (off0,off1,off2,len0,len1,len2) -> uint8[n,32]."""
        buf = np.ascontiguousarray(np.frombuffer(buf, np.uint8) if isinstance(buf, (bytes, bytearray)) else buf)
        jobs = np.ascontiguousarray(jobs, dtype=np.uint32).reshape(-1, 6)
        out = np.zeros((jobs.shape[0], 32), np.uint8)
        self._ck(lib().fabgpu_sha256_segments(self._h, _p(buf), ctypes.c_size_t(buf.shape[0]), _p(jobs), ctypes.c_size_t(jobs.shape[0]), _p(out)))
        return out

    def last_timing(self):
        """[key lookup, host gates, device, scatter] microseconds of the last bccsp_verify_batch call."""
        out = (ctypes.c_double * 4)()
        self._ck(lib().fabgpu_last_timing(self._h, out))
        return [float(x) for x in out]

    # ---- test hooks -------------------------------------------------------------------------------------
    def test_fieldop(self, op, a, b):
        a = np.ascontiguousarray(a, dtype=np.uint8).reshape(-1, 32)
        b = np.ascontiguousarray(b, dtype=np.uint8).reshape(-1, 32)
        out = np.zeros_like(a)
        self._ck(lib().fabgpu_test_fieldop(self._h, ctypes.c_int(op), _p(a), _p(b), ctypes.c_size_t(a.shape[0]), _p(out)))
        return out

    def test_table_entries(self, key_slot, window, digit):
        """Sampled table entries -> (n, 16) little-endian u32 limbs, X then Y, Montgomery form.  key_slot -1: the generator table;
        >= 0: the window table in that raw key slot; <= -2: the small table of that keys_register_small handle (FabGpuError if stale)."""
        window = np.ascontiguousarray(window, dtype=np.uint32)
        digit = np.ascontiguousarray(digit, dtype=np.uint32)
        out = np.zeros((window.shape[0], 64), np.uint8)
        self._ck(lib().fabgpu_test_table_entries(self._h, ctypes.c_int(key_slot), _p(window), _p(digit), ctypes.c_size_t(window.shape[0]), _p(out)))
        return out.view("<u4").reshape(-1, 16)
