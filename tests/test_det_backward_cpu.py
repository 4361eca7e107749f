"""CPU: the deterministic-backward C ABI (gpsg_rasterize_backward*_ex) and its Python switch -- workspace sizes, argument
validation and the torch.use_deterministic_algorithms helper.  No call here reaches the device."""
import ctypes as C

import pytest
import torch

DET = 1   # GPSG_BWD_DETERMINISTIC
SIZES = [(0, 0), (1, 0), (1, 1), (7, 3), (1000, 5000), (499_400, 1_307_000), (262_144, 4_100_000), (2_000_000, 30_000_000)]


def test_flag_zero_sizes_equal_the_old_entry_points(built_lib):
    from gps_gaussian_b200 import _lib
    L = _lib.lib
    assert _lib.BWD_DETERMINISTIC == DET
    for P, N in SIZES:
        assert L.gpsg_rasterize_backward_workspace_bytes_ex(P, N, 0) == L.gpsg_rasterize_backward_workspace_bytes(P)
        assert L.gpsg_rasterize_backward_maps_workspace_bytes_ex(P, N, 0) == L.gpsg_rasterize_backward_maps_workspace_bytes(P)
    assert L.gpsg_rasterize_backward_workspace_bytes_ex(-5, 0, 0) == L.gpsg_rasterize_backward_workspace_bytes(-5)


def test_deterministic_workspace_stays_within_320_bytes_per_pair(built_lib):
    """DET adds a 1-byte slot mask and 8 slots x 9 floats per (tile, Gaussian) pair: 289 B plus alignment, <= 320 B."""
    from gps_gaussian_b200 import _lib
    L = _lib.lib
    for P, N in SIZES:
        for det_fn, base_fn in ((L.gpsg_rasterize_backward_workspace_bytes_ex, L.gpsg_rasterize_backward_workspace_bytes),
                                (L.gpsg_rasterize_backward_maps_workspace_bytes_ex, L.gpsg_rasterize_backward_maps_workspace_bytes)):
            extra = det_fn(P, N, DET) - base_fn(P)
            assert 289 * N <= extra <= 320 * N + 512, (P, N, extra)
    # C2 (P = 499 400, N ~ 1.307 M pairs): 0.378 GB of DET scratch on top of the 30 MB of the default workspace
    extra = L.gpsg_rasterize_backward_workspace_bytes_ex(499_400, 1_307_000, DET) - L.gpsg_rasterize_backward_workspace_bytes(499_400)
    assert extra < 0.38e9


def test_ex_argument_validation_without_gpu(built_lib):
    from gps_gaussian_b200 import _lib
    L = _lib.lib
    s = _lib.RasterSettings()
    s.image_height, s.image_width = 16, 16
    nul = [None] * 21
    # unknown flag bits: refused before anything else is looked at
    for flags in (2, 4, -1, 1 | 8):
        assert L.gpsg_rasterize_backward_ex(C.byref(s), 0, None, 10, 0, 5, *nul, flags) == -1
        assert b"flag" in L.gpsg_last_error()
        assert L.gpsg_rasterize_backward_maps_ex(C.byref(s), 0, None, 8, 5, *([None] * 6), *([None] * 5), *([None] * 5),
                                                 None, flags) == -1
        assert b"flag" in L.gpsg_last_error()
        assert L.gpsg_rasterize_backward_workspace_bytes_ex(10, 5, flags) == 0
        assert L.gpsg_rasterize_backward_maps_workspace_bytes_ex(10, 5, flags) == 0
    assert L.gpsg_rasterize_backward_workspace_bytes_ex(10, -1, DET) == 0          # a pair count the mode cannot size
    # NULL pointers with valid flags, in both modes
    for flags in (0, DET):
        assert L.gpsg_rasterize_backward_ex(None, 0, None, 10, 0, 5, *nul, flags) == -1
        assert b"settings is NULL" in L.gpsg_last_error()
        assert L.gpsg_rasterize_backward_ex(C.byref(s), 0, None, 10, 0, 5, *nul, flags) == -1
        assert b"NULL" in L.gpsg_last_error()
        assert L.gpsg_rasterize_backward_ex(C.byref(s), 0, None, -1, 0, 5, *nul, flags) == -1
        assert L.gpsg_rasterize_backward_maps_ex(C.byref(s), 0, None, 8, 5, *([None] * 6), *([None] * 5), *([None] * 5),
                                                 None, flags) == -1
        assert b"NULL" in L.gpsg_last_error()
        assert L.gpsg_rasterize_backward_ex(C.byref(s), 0, None, 0, 0, 0, *nul, flags) == 0    # P = 0: nothing to do


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
