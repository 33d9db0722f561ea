"""Error contract of the C ABI (include/pnr.h): invalid arguments are rejected with a negative return code and a
message in pnr_last_error() BEFORE any CUDA call, so this runs without a GPU (no compute is launched).
Mirrors the reference's behaviour of asserting / raising on malformed inputs (e.g. nerf.py:268 `assert len(rays.shape) == 3`)."""
import ctypes as C
import os

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "pixel-nerf_b200", "lib", "libpnr_sm90.so")


@pytest.fixture(scope="module")
def lib():
    if not os.path.exists(LIB):
        import __graft_entry__ as ge
        ge.build()
    L = C.CDLL(LIB)
    L.pnr_last_error.restype = C.c_char_p
    i32, i64, vp, f32 = C.c_int32, C.c_int64, C.c_void_p, C.c_float
    L.pnr_gen_rays.argtypes = [vp, i64, i32, i32, f32, f32, f32, f32, f32, f32, i64, i64, vp, vp]
    L.pnr_frames_u8.argtypes = [vp, i64, vp, vp]
    L.pnr_sample_coarse.argtypes = [vp, vp, vp, vp, i64, i32, vp]
    L.pnr_composite.argtypes = [vp, vp, vp, i32, vp, vp, vp, i64, i32, vp]
    L.pnr_sample_fine.argtypes = [vp, vp, vp, vp, vp, vp, vp, f32, vp, i64, i32, i32, i32, vp]
    L.pnr_pack_latent.argtypes = [vp, vp, i32, i32, i32, i32, vp]
    L.pnr_render.argtypes = [vp, vp, vp, vp, vp, vp, vp, i64, vp, C.c_size_t, vp]
    L.pnr_field_eval.argtypes = [vp, vp, vp, vp, vp, i64, i32, vp, C.c_size_t, vp]
    for n in ("pnr_gen_rays", "pnr_frames_u8", "pnr_sample_coarse", "pnr_composite", "pnr_sample_fine",
              "pnr_pack_latent", "pnr_render", "pnr_field_eval"):
        getattr(L, n).restype = C.c_int
    return L


def rejected(lib, rc, needle):
    msg = lib.pnr_last_error().decode()
    return rc < 0 and needle in msg


FAKE = 0x1000   # never dereferenced: every call below must fail (or return) before touching memory or CUDA


def test_gen_rays_rejects_bad_ranges(lib):
    assert rejected(lib, lib.pnr_gen_rays(FAKE, 2, 4, 3, 1.0, 1.0, 2.0, 1.5, 0.1, 1.0, 20, 8, FAKE, None), "outside the pixel grid")
    assert rejected(lib, lib.pnr_gen_rays(FAKE, 2, 4, 3, 1.0, 1.0, 2.0, 1.5, 0.1, 1.0, -1, 4, FAKE, None), "outside the pixel grid")
    assert rejected(lib, lib.pnr_gen_rays(FAKE, 2, 0, 3, 1.0, 1.0, 2.0, 1.5, 0.1, 1.0, 0, 0, FAKE, None), "bad sizes")
    assert rejected(lib, lib.pnr_gen_rays(None, 2, 4, 3, 1.0, 1.0, 2.0, 1.5, 0.1, 1.0, 0, 4, FAKE, None), "NULL")
    assert rejected(lib, lib.pnr_gen_rays(FAKE, 2, 4, 3, 0.0, 1.0, 2.0, 1.5, 0.1, 1.0, 0, 4, FAKE, None), "zero focal")
    assert rejected(lib, lib.pnr_gen_rays(FAKE, 2, 4, 3, 1.0, 1.0, 2.0, 1.5, 0.1, 1.0, 0, 4, FAKE + 4, None), "aligned")
    assert lib.pnr_gen_rays(None, 2, 4, 3, 1.0, 1.0, 2.0, 1.5, 0.1, 1.0, 5, 0, None, None) == 0   # empty range: no-op


def test_frames_u8_rejects_bad_arguments(lib):
    assert rejected(lib, lib.pnr_frames_u8(FAKE, -1, FAKE, None), "bad size")
    assert rejected(lib, lib.pnr_frames_u8(None, 4, FAKE, None), "NULL")
    assert rejected(lib, lib.pnr_frames_u8(FAKE + 4, 4, FAKE, None), "aligned")
    assert lib.pnr_frames_u8(None, 0, None, None) == 0


def test_stage_entries_reject_bad_sizes_and_null(lib):
    assert rejected(lib, lib.pnr_sample_coarse(FAKE, None, FAKE, FAKE, 4, 0, None), "bad sizes")
    assert rejected(lib, lib.pnr_sample_coarse(None, None, FAKE, FAKE, 4, 8, None), "NULL")
    assert lib.pnr_sample_coarse(None, None, None, None, 0, 8, None) == 0                       # empty batch
    assert rejected(lib, lib.pnr_composite(FAKE, FAKE, FAKE, 1, None, FAKE, FAKE, 4, 0, None), "bad sizes")
    assert rejected(lib, lib.pnr_composite(FAKE, FAKE, None, 1, None, FAKE, FAKE, 4, 8, None), "NULL")
    assert rejected(lib, lib.pnr_sample_fine(FAKE, FAKE, FAKE, FAKE, FAKE, FAKE, FAKE, 0.01, FAKE, 4, 8, 4, 5, None), "bad sizes")
    assert rejected(lib, lib.pnr_sample_fine(FAKE, FAKE, None, FAKE, FAKE, FAKE, FAKE, 0.01, FAKE, 4, 8, 4, 2, None), "importance")
    assert rejected(lib, lib.pnr_sample_fine(FAKE, FAKE, FAKE, None, FAKE, FAKE, FAKE, 0.01, FAKE, 4, 8, 4, 2, None), "depth")
    assert rejected(lib, lib.pnr_pack_latent(None, FAKE, 1, 512, 8, 8, None), "NULL")
    assert rejected(lib, lib.pnr_pack_latent(FAKE, FAKE, 1, 512, 0, 8, None), "bad latent shape")


def test_render_and_field_reject_null_descriptors(lib):
    assert rejected(lib, lib.pnr_render(None, None, None, None, FAKE, None, None, 4, FAKE, 1024, None), "NULL")
    assert rejected(lib, lib.pnr_field_eval(None, None, FAKE, FAKE, FAKE, 4, 0, FAKE, 1024, None), "NULL")
