"""fabgpu_block_pvt_updates is exported with the header's record layout, and refuses a NULL context without a device."""
import ctypes
import os
import re

from util import ROOT, pkg


def test_symbol_exported_and_null_context_refused():
    B = pkg().binding
    L = ctypes.CDLL(B.LIB_PATH)
    assert hasattr(L, "fabgpu_block_pvt_updates") and "fabgpu_block_pvt_updates" in B.EXPORTS
    hdr = open(os.path.join(ROOT, "include", "fabgpu_ecdsa.h")).read()
    assert int(re.search(r"#define FABGPU_PVT_UPDATE_WORDS (\d+)", hdr).group(1)) == B.PVT_UPDATE_WORDS
    assert int(re.search(r"#define FABGPU_UPDATE_RENEW (\d+)", hdr).group(1)) == B.UPDATE_RENEW
    n, complete = ctypes.c_size_t(0), ctypes.c_int(0)
    out = (ctypes.c_int32 * 4)()
    rc = L.fabgpu_block_pvt_updates(None, 0, ctypes.c_uint64(1), None, None, None, ctypes.c_size_t(0), None, out, None, ctypes.c_size_t(0),
                                    ctypes.byref(n), ctypes.byref(complete))
    assert rc == B.E_ARG
