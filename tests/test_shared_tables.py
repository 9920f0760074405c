"""No GPU: fabgpu_init_shared is exported and declared, and refuses a missing context before it looks for a device."""
import ctypes

import pytest

from util import pkg


def test_init_shared_is_exported():
    b = pkg().binding
    assert "fabgpu_init_shared" in b.EXPORTS
    assert hasattr(ctypes.CDLL(b.LIB_PATH), "fabgpu_init_shared")


def test_init_shared_without_a_context_is_refused():
    b = pkg().binding
    L = b.lib()
    out = ctypes.c_void_p(0x1234)
    assert L.fabgpu_init_shared(None, ctypes.c_size_t(64), ctypes.byref(out)) == b.E_ARG
    assert out.value is None
    assert b"share" in L.fabgpu_last_error(None)
    assert L.fabgpu_init_shared(None, ctypes.c_size_t(64), None) == b.E_ARG


def test_binding_refuses_a_closed_context_and_device_ids():
    b = pkg().binding

    class Closed:
        _h = ctypes.c_void_p()

    with pytest.raises(b.FabGpuError) as ei:
        b.Context(max_batch=64, share_tables_with=Closed())
    assert ei.value.code == b.E_ARG
    with pytest.raises(ValueError):
        b.Context(max_batch=64, device_ids=[0], share_tables_with=Closed())
