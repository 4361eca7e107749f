"""CPU: the deterministic-backward C ABI (the `flags` word of gpsg_rasterize_backward / _maps and their workspace-size
queries) and its Python switch -- workspace sizes, argument validation and the torch.use_deterministic_algorithms helper.
No call here reaches the device."""
import ctypes as C

import pytest
import torch

DET = 1   # GPSG_BWD_DETERMINISTIC
SIZES = [(0, 0), (1, 0), (1, 1), (7, 3), (1000, 5000), (499_400, 1_307_000), (262_144, 4_100_000), (2_000_000, 30_000_000)]


def _size_queries(L):
    return L.gpsg_rasterize_backward_workspace_bytes, L.gpsg_rasterize_backward_maps_workspace_bytes


def test_flag_zero_sizes_depend_on_neither_pairs_nor_aux(built_lib):
    """Without GPSG_BWD_DETERMINISTIC the workspace size depends on neither the pair count nor aux."""
    from gps_gaussian_b200 import _lib
    L = _lib.lib
    assert _lib.BWD_DETERMINISTIC == DET
    for ws in _size_queries(L):
        for P, N in SIZES:
            for aux in (0, 1):
                assert ws(P, N, 0, aux) == ws(P, 0, 0, 0), (ws.__name__, P, N, aux)
    assert L.gpsg_rasterize_backward_workspace_bytes(-5, 0, 0, 0) == L.gpsg_rasterize_backward_workspace_bytes(1, 0, 0, 0)


def test_deterministic_workspace_stays_within_320_bytes_per_pair(built_lib):
    """DET adds a 1-byte slot mask and 8 slots x 9 floats per (tile, Gaussian) pair: 289 B plus alignment, <= 320 B."""
    from gps_gaussian_b200 import _lib
    L = _lib.lib
    for ws in _size_queries(L):
        for P, N in SIZES:
            extra = ws(P, N, DET, 0) - ws(P, 0, 0, 0)
            assert 289 * N <= extra <= 320 * N + 512, (ws.__name__, P, N, extra)
    # C2 (P = 499 400, N ~ 1.307 M pairs): 0.378 GB of DET scratch on top of the 30 MB of the default workspace
    ws = L.gpsg_rasterize_backward_workspace_bytes
    extra = ws(499_400, 1_307_000, DET, 0) - ws(499_400, 0, 0, 0)
    assert extra < 0.38e9


def test_backward_flags_argument_validation_without_gpu(built_lib):
    from gps_gaussian_b200 import _lib
    L = _lib.lib
    s = _lib.RasterSettings()
    s.image_height, s.image_width = 16, 16
    nul = [None] * 23
    maps_nul = [None] * 19
    # unknown flag bits: refused before anything else is looked at
    for flags in (2, 4, -1, 1 | 8):
        assert L.gpsg_rasterize_backward(C.byref(s), 0, None, 10, 0, 5, *nul, flags) == -1
        assert b"flag" in L.gpsg_last_error()
        assert L.gpsg_rasterize_backward_maps(C.byref(s), 0, None, 8, 5, *maps_nul, flags) == -1
        assert b"flag" in L.gpsg_last_error()
        for ws in _size_queries(L):
            assert ws(10, 5, flags, 0) == 0
            assert b"flag" in L.gpsg_last_error()
    for ws in _size_queries(L):
        assert ws(10, -1, DET, 0) == 0                                          # a pair count the mode cannot size
        assert b"num_rendered" in L.gpsg_last_error()
        for aux in (2, -1):                                                     # aux is 0 or 1, in both modes
            for flags in (0, DET):
                assert ws(10, 5, flags, aux) == 0
                assert b"aux" in L.gpsg_last_error()
    # NULL pointers with valid flags, in both modes
    for flags in (0, DET):
        assert L.gpsg_rasterize_backward(None, 0, None, 10, 0, 5, *nul, flags) == -1
        assert b"settings is NULL" in L.gpsg_last_error()
        assert L.gpsg_rasterize_backward(C.byref(s), 0, None, 10, 0, 5, *nul, flags) == -1
        assert b"NULL" in L.gpsg_last_error()
        assert L.gpsg_rasterize_backward(C.byref(s), 0, None, -1, 0, 5, *nul, flags) == -1
        assert L.gpsg_rasterize_backward_maps(C.byref(s), 0, None, 8, 5, *maps_nul, flags) == -1
        assert b"NULL" in L.gpsg_last_error()
        assert L.gpsg_rasterize_backward(C.byref(s), 0, None, 0, 0, 0, *nul, flags) == 0    # P = 0: nothing to do


def test_backward_flags_follow_torch_determinism_switch(built_lib):
    from gps_gaussian_b200 import _lib
    was, warn = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
    try:
        torch.use_deterministic_algorithms(False)
        assert _lib.backward_flags() == 0 and _lib.backward_flags(None) == 0
        assert _lib.backward_flags(True) == DET
        torch.use_deterministic_algorithms(True)
        assert _lib.backward_flags() == DET
        assert _lib.backward_flags(False) == 0                                   # an explicit argument wins
        torch.use_deterministic_algorithms(True, warn_only=True)
        assert _lib.backward_flags() == DET
    finally:
        torch.use_deterministic_algorithms(was, warn_only=warn)
    assert torch.are_deterministic_algorithms_enabled() == was
