"""Stage-1 preview splat without a GPU: the C ABI's exports, workspace size and refusals, the serial reference it is
checked against (tests/splat_reference.py) on hand-made cases, and the `taichi` stand-in with the unmodified reference
lib/TaichiRender.py (when the original project is staged)."""
import ctypes as C
import inspect

import numpy as np
import pytest

from splat_reference import fresh_buffers, saturating_pixel, splat_serial


def _lib(built_lib):
    from gps_gaussian_b200 import _lib
    return _lib


def test_abi_exports_and_workspace(built_lib):
    L = _lib(built_lib)
    for name in ("gpsg_point_splat_workspace_bytes", "gpsg_point_splat"):
        assert name in L.EXPORTED and hasattr(C.CDLL(built_lib), name)
    ws = L.lib.gpsg_point_splat_workspace_bytes
    assert ws(1, 1) == 12 and ws(2, 1024) == 2 * 1024 * 1024 * 12     # u64 key + u32 first-zero index per pixel
    assert ws(0, 8) == 0 and ws(2, 0) == 0 and ws(-1, 8) == 0 and ws(1, 46341) == 0   # 46341^2 >= 2^31
    assert L.lib.gpsg_version() == 90


@pytest.mark.parametrize("args, msg", [
    ((-1, 4, 8, 4), "negative size"),
    ((1, -4, 8, 4), "negative size"),
    ((1, 4, 8, -4), "negative size"),
    ((1, 4, 0, 4), "res must be >= 1"),
    ((0, 0, 0, 0), "res must be >= 1"),
    ((1, 5, 8, 4), "N > rows_per_batch"),
    ((1, 4, 46341, 4), "res^2 must be < 2^31"),
])
def test_abi_refusals(built_lib, args, msg):
    L = _lib(built_lib)
    B, N, res, rows = args
    rc = L.lib.gpsg_point_splat(0, None, B, N, res, rows, None, None, None, None, None)
    assert rc == -1 and msg in L.lib.gpsg_last_error().decode()


def test_abi_null_pointers_and_noops(built_lib):
    L = _lib(built_lib)
    f = L.lib.gpsg_point_splat
    buf = (C.c_float * 64)()
    ptrs = [C.cast(buf, C.c_void_p)] * 5
    for k in range(5):
        args = list(ptrs)
        args[k] = None
        assert f(0, None, 1, 4, 8, 4, *args) == -1 and "NULL pointer" in L.lib.gpsg_last_error().decode()
    # no work: no pointer is needed and nothing touches a device
    assert f(0, None, 0, 4, 8, 4, None, None, None, None, None) == 0
    assert f(0, None, 2, 0, 8, 0, None, None, None, None, None) == 0


# ---- the serial reference -----------------------------------------------------------------------------------------

def _pts(rows):
    return np.array([rows], np.float32)


def test_reference_saturating_cast():
    x = np.array([np.nan, -np.nan, 1e10, -1e10, np.inf, -np.inf, 2.0 ** 31, -0.9, 0.9, 3.99, 7.0, 8.0, -0.0], np.float32)
    assert saturating_pixel(x, 8).tolist() == [0, 0, 7, 0, 7, 0, 7, 0, 0, 3, 7, 7, 0]
    pts = _pts([[1e10, -1e10, 0.5, 1, 2, 3], [np.nan, 1e10, 0.25, 4, 5, 6], [-1e10, np.nan, 0.75, 7, 8, 9]])
    depth, color = fresh_buffers(1, 8)
    splat_serial(pts, np.ones((1, 3), np.float32), depth, color)
    assert depth[0, 0, 0, 7] == np.float32(0.5) and color[0, :, 0, 7].tolist() == [1, 2, 3]
    assert depth[0, 0, 7, 0] == np.float32(0.25) and color[0, :, 7, 0].tolist() == [4, 5, 6]
    assert depth[0, 0, 0, 0] == np.float32(0.75) and color[0, :, 0, 0].tolist() == [7, 8, 9]


def test_reference_ties():
    # within one call the highest index wins; across calls the second call wins (z >= old)
    depth, color = fresh_buffers(1, 4)
    splat_serial(_pts([[1, 1, 0.5, 1, 0, 0], [1.5, 1.2, 0.5, 0, 1, 0], [1.9, 1.9, 0.25, 0, 0, 1]]), np.ones((1, 3)), depth, color)
    assert depth[0, 0, 1, 1] == np.float32(0.5) and color[0, :, 1, 1].tolist() == [0, 1, 0]
    splat_serial(_pts([[1, 1, 0.5, 9, 9, 9], [1, 1, 0.125, 8, 8, 8]]), np.ones((1, 2)), depth, color)
    assert depth[0, 0, 1, 1] == np.float32(0.5) and color[0, :, 1, 1].tolist() == [9, 9, 9]
    # a nearer point earlier in the call still beats a farther later one
    depth, color = fresh_buffers(1, 4)
    splat_serial(_pts([[2, 2, 0.9, 1, 1, 1], [2, 2, 0.3, 2, 2, 2]]), np.ones((1, 2)), depth, color)
    assert depth[0, 0, 2, 2] == np.float32(0.9) and color[0, :, 2, 2].tolist() == [1, 1, 1]


def test_reference_signed_zero_and_negative_z():
    # -0 and +0 tie: colour from the last, depth keeps the first strictly greater write
    depth, color = fresh_buffers(1, 4)
    splat_serial(_pts([[0, 0, -0.0, 1, 1, 1], [0, 0, 0.0, 2, 2, 2], [0, 0, -0.0, 3, 3, 3]]), np.ones((1, 3)), depth, color)
    assert color[0, :, 0, 0].tolist() == [3, 3, 3] and not np.signbit(depth[0, 0, 0, 0])
    depth[...] = -1.0
    splat_serial(_pts([[0, 0, -0.0, 4, 4, 4], [0, 0, 0.0, 5, 5, 5]]), np.ones((1, 2)), depth, color)
    assert color[0, :, 0, 0].tolist() == [5, 5, 5] and depth[0, 0, 0, 0] == 0 and np.signbit(depth[0, 0, 0, 0])
    # negative z never draws on the initial depth of 0
    depth, color = fresh_buffers(1, 4)
    splat_serial(_pts([[3, 3, -0.5, 1, 1, 1], [3, 3, -np.inf, 1, 1, 1]]), np.ones((1, 2)), depth, color)
    assert depth[0, 0, 3, 3] == 0 and color[0, :, 3, 3].tolist() == [-1, -1, -1]


def test_reference_nan_and_mask():
    depth, color = fresh_buffers(1, 4)
    pts = _pts([[1, 1, np.nan, 1, 1, 1], [2, 2, 0.5, 2, 2, 2], [3, 3, 0.5, 3, 3, 3], [0, 3, 0.5, 4, 4, 4]])
    mask = np.array([[1, np.nan, 0.49, 0.5]], np.float32)
    splat_serial(pts, mask, depth, color)
    assert depth[0, 0, 1, 1] == 0 and color[0, 0, 1, 1] == -1                       # NaN z: skipped
    assert depth[0, 0, 2, 2] == np.float32(0.5) and color[0, 0, 2, 2] == 2          # NaN mask: not < 0.5, drawn
    assert depth[0, 0, 3, 3] == 0 and color[0, 0, 3, 3] == -1                       # mask 0.49: skipped
    assert depth[0, 0, 3, 0] == np.float32(0.5) and color[0, 0, 3, 0] == 4          # mask 0.5: drawn


def test_reference_loop_domain():
    pts = np.tile(_pts([[1, 1, 0.5, 1, 1, 1], [2, 2, 0.5, 2, 2, 2]]), (2, 1, 1))
    depth, color = fresh_buffers(2, 4)
    splat_serial(pts, np.ones((2, 2, 1)), depth, color, B=1, N=1)
    assert color[0, 0, 1, 1] == 1 and color[0, 0, 2, 2] == -1                        # row 1 is outside N
    assert (depth[1] == 0).all() and (color[1] == -1).all()                          # batch 1 is outside B


def test_reference_matches_oracle_default_form():
    """On inputs where C's cast is defined, one call on fresh buffers is the oracle's own `taichi_splat`."""
    from oracle.raster_oracle import taichi_splat
    rng = np.random.default_rng(3)
    pts = np.concatenate([rng.uniform(-4, 36, (2, 3000, 2)), rng.integers(1, 5, (2, 3000, 1)) / 4,
                          rng.uniform(0, 1, (2, 3000, 3))], 2).astype(np.float32)
    mask = (rng.uniform(size=(2, 3000)) > 0.2).astype(np.float32)
    want_d, want_c = taichi_splat(pts, mask, 32)
    depth, color = fresh_buffers(2, 32)
    splat_serial(pts, mask, depth, color)
    assert depth.tobytes() == want_d.tobytes() and color.tobytes() == want_c.tobytes()


# ---- the `taichi` stand-in with the unmodified reference --------------------------------------------------------------

def _staged():
    from gps_gaussian_b200 import harness
    return harness.staged_reference()


needs_ref = pytest.mark.skipif(_staged() is None, reason="oracle/_ref not staged (run __graft_entry__.build() where the "
                                                         "original project is checked out)")


@pytest.fixture(scope="module")
def taichi_render(built_lib):
    from gps_gaussian_b200 import harness
    harness.add_reference_to_path()
    import lib.TaichiRender as TR
    return TR


@needs_ref
def test_standin_imports_unmodified_reference(taichi_render):
    import os
    import taichi
    from gps_gaussian_b200 import harness
    assert "gps-gaussian_b200" in taichi.__file__
    assert taichi_render.__file__.startswith(harness.REF_STAGED)
    r = taichi_render.TaichiRenderBatch(bs=1, res=16)
    assert r.res == 16 and r.coord.shape == (1, 256)
    fn = taichi_render.TaichiRenderBatch.render_respective_color
    assert taichi.kernel_digest(fn.__wrapped__) == taichi._SPLAT_DIGEST
    assert fn.__qualname__ == "TaichiRenderBatch.render_respective_color"
    with open(os.path.join(harness.REF_STAGED, "lib", "TaichiRender.py"), "rb") as a:
        assert b"import taichi as ti" in a.read()


@needs_ref
def test_standin_refuses_cpu_tensors(taichi_render):
    import torch
    r = taichi_render.TaichiRenderBatch(bs=1, res=4)
    args = (torch.zeros(1, 16, 6), torch.ones(1, 16, 1), torch.zeros(1, 1, 4, 4), torch.zeros(1, 3, 4, 4))
    with pytest.raises(TypeError, match="must be a CUDA float32 torch tensor"):
        r.render_respective_color(*args)
    with pytest.raises(TypeError, match="must be a CUDA float32 torch tensor"):
        r.render_respective_color(args[0].double(), *args[1:])


@needs_ref
def test_standin_refuses_altered_kernel(taichi_render, tmp_path):
    import importlib.util
    import taichi as ti
    with open(taichi_render.__file__) as f:
        src = f.read()
    assert "pts[B, i, 2] >= ti.atomic_max" in src
    edits = {"body": src.replace("pts_mask[B, i, 0] < 0.5", "pts_mask[B, i, 0] < 0.25"),      # same name, edited body
             "name": src.replace("def render_respective_color", "def render_other"),         # same body, another name
             "spaces": src.replace("IX = ti.min(", "IX  =  ti.min(")}                          # whitespace only
    for what, edited in edits.items():
        path = tmp_path / f"edited_{what}.py"
        path.write_text(edited)
        spec = importlib.util.spec_from_file_location(f"edited_{what}", path)
        mod = importlib.util.module_from_spec(spec)
        spec.loader.exec_module(mod)
        r = mod.TaichiRenderBatch(bs=1, res=4)
        fn = getattr(r, "render_respective_color", None) or r.render_other
        if what == "spaces":                            # recognised: gets as far as the tensor checks
            with pytest.raises(TypeError, match="CUDA float32"):
                fn(None, None, None, None)
            continue
        with pytest.raises(NotImplementedError, match="taichi stand-in"):
            fn(None, None, None, None)

    @ti.kernel
    def other(x: ti.types.ndarray()):
        pass
    with pytest.raises(NotImplementedError, match="is not supported"):
        other(None)
