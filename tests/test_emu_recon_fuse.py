"""pnr_tsdf_fuse (csrc/pnr_recon.cu) on the host emulator (built by tests/recon_emu.py): the fused volume bit for bit
against the numpy oracle (oracle/pnr_recon_fuse.py) on the analytic sphere and on random maps with every branch of the
rule -- opacity below and exactly at min_opacity, voxels behind a camera and outside its image, projections on a
rounding tie, a non-square image with an off-centre principal point -- and the error codes."""
import ctypes as C

import numpy as np
import pytest
import torch

import emu_util as eu
import recon_emu
from fuse_util import fuse, sphere_maps, views

PNR_ERR_INVALID = -1


def emu_fuse(depth, opacity, poses, fx, fy, cx, cy, lo, hi, reso, trunc, min_opacity):
    depth = torch.from_numpy(np.ascontiguousarray(depth, dtype=np.float32))
    opacity = torch.from_numpy(np.ascontiguousarray(opacity, dtype=np.float32))
    poses = torch.from_numpy(np.ascontiguousarray(poses, dtype=np.float32))
    V, H, W = depth.shape
    out = torch.full(tuple(reso), 7.0)
    rc = recon_emu.lib().pnr_tsdf_fuse(eu.ptr(depth), eu.ptr(opacity), V, W, H, eu.ptr(poses), fx, fy, cx, cy,
                                       (C.c_double * 3)(*lo), (C.c_double * 3)(*hi), (C.c_int32 * 3)(*reso), trunc,
                                       min_opacity, eu.ptr(out), None)
    assert rc == 0, recon_emu.lib().pnr_last_error().decode()
    return out.numpy()


def assert_same(*args):
    got = emu_fuse(*args)
    want = fuse.tsdf_fuse(*args)
    assert got.shape == want.shape
    assert np.array_equal(got.view(np.int32), want.view(np.int32))
    return got


def test_sphere():
    poses = views(6, 3.0)
    depth, opacity = sphere_maps(poses, 40, 40, 70.0, 0.5)
    t = assert_same(depth, opacity, poses.numpy(), 70.0, 70.0, 20.0, 20.0, (-0.8,) * 3, (0.8,) * 3, (17, 15, 16),
                    0.2, 0.5)
    assert (t < 0).any() and (t > 0).any() and (t == -1).any() and (t == 1).any()


def random_case(seed, V=5, W=11, H=7):
    g = np.random.default_rng(seed)
    import util
    poses = torch.stack([util.pose_spherical(float(g.uniform(-180, 180)), float(g.uniform(-80, 80)),
                                             float(g.uniform(0.3, 2.0))) for _ in range(V)]).numpy()
    poses[:, :3, 3] += g.uniform(-0.3, 0.3, (V, 3)).astype(np.float32)   # some cameras inside the box
    opacity = g.choice(np.float32([0.0, 0.2, 0.4999999, 0.5, 0.5000001, 0.8, 1.0]), size=(V, H, W))
    depth = (opacity * g.uniform(0.0, 3.0, (V, H, W))).astype(np.float32)
    return poses, depth, opacity


@pytest.mark.parametrize("seed", range(4))
def test_random_maps(seed):
    poses, depth, opacity = random_case(seed)
    V, H, W = depth.shape
    t = assert_same(depth, opacity, poses, 6.0, 5.5, 6.3, 2.75, (-1.0, -0.9, -1.1), (1.0, 1.2, 0.8), (9, 8, 7),
                    0.25, 0.5)
    assert (t == 1).any() and (t == -1).any() and ((t > -1) & (t < 1)).any()


def test_rounding_ties_and_visibility():
    """A camera at z = 3 looking down -z with fx = 3: voxel x of the plane z = 0 projects to cx + x, so the grid's
    half-integer x land exactly on ties; voxels above z = 3 are behind the camera, those with |x| large outside."""
    P = np.eye(4, dtype=np.float32)
    P[2, 3] = 3.0
    g = np.random.default_rng(5)
    W, H = 6, 5
    opacity = g.choice(np.float32([0.0, 0.5, 1.0]), size=(1, H, W))
    depth = (opacity * g.uniform(1.0, 4.0, (1, H, W))).astype(np.float32)
    args = (depth, opacity, P[None], 3.0, 3.0, 2.0, 2.0)
    assert_same(*args, (-3.0, -3.0, 0.0), (3.0, 3.0, 0.0), (13, 13, 1), 0.5, 0.5)       # x, y in steps of 0.5
    t = assert_same(*args, (-1.0, -1.0, 2.0), (1.0, 1.0, 4.0), (5, 5, 9), 0.5, 0.5)       # z across the camera
    assert (t[:, :, -4:] == 1.0).all()                                                     # z >= 3: nobody sees them
    # the same through a non-square image with an off-centre principal point and unequal focals
    assert_same(depth, opacity, P[None], 2.0, 4.0, 1.0, 3.0, (-2.5, -2.0, -0.5), (2.5, 2.0, 0.5), (11, 9, 3), 0.3, 1.0)


def test_error_codes():
    L = recon_emu.lib()
    depth = torch.ones(1, 3, 4)
    poses = torch.eye(4)[None].contiguous()
    out = torch.empty(2, 2, 2)
    lo, hi = (C.c_double * 3)(-1, -1, -1), (C.c_double * 3)(1, 1, 1)

    def call(d=eu.ptr(depth), o=eu.ptr(depth), V=1, W=4, H=3, p=eu.ptr(poses), lo=lo, hi=hi,
             reso=(C.c_int32 * 3)(2, 2, 2), trunc=0.1, m=0.5, t=eu.ptr(out)):
        return L.pnr_tsdf_fuse(d, o, V, W, H, p, 1.0, 1.0, 2.0, 1.5, lo, hi, reso, trunc, m, t, None)
    assert call() == 0
    for kw in (dict(d=None), dict(o=None), dict(p=None), dict(t=None), dict(lo=None), dict(hi=None), dict(reso=None),
               dict(V=0), dict(W=0), dict(H=-1), dict(reso=(C.c_int32 * 3)(2, 0, 2)),
               dict(reso=(C.c_int32 * 3)(4096, 4096, 8192)), dict(trunc=0.0), dict(trunc=-1.0),
               dict(trunc=float("nan")), dict(trunc=float("inf")), dict(m=0.0), dict(m=1.0000001),
               dict(m=float("nan"))):
        assert call(**kw) == PNR_ERR_INVALID, kw
    assert call(m=1.0) == 0
