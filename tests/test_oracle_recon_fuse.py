"""The TSDF fusion rule (oracle/pnr_recon_fuse.py, the restatement pnr_tsdf_fuse is compared against) on analytic
scenes: the depth maps of a sphere from a turntable plus a top and a bottom view fuse into a volume whose marching
cubes is one closed, consistently oriented sphere within a voxel of the true radius; and the classification cases one
by one (background carves, the occluded interior is inside, a voxel no camera sees is outside)."""
import numpy as np
import torch

from fuse_util import fuse, index_to_world, sphere_maps, views
from recon_util import recon

LO, HI, RESO = (-1.0, -1.0, -1.0), (1.0, 1.0, 1.0), (48, 48, 48)
W = H = 96
FOCAL = 160.0
R = 0.5


def default_trunc(lo, hi, reso):
    """fuse_views' default: 3 voxel diagonals of the coarsest axis."""
    return 3.0 * np.sqrt(3.0) * float(np.abs((np.array(hi) - np.array(lo)) / (np.array(reso) - 1)).max())


def sphere_tsdf(n_turn=16, reso=RESO):
    poses = views(n_turn, 3.0)
    depth, opacity = sphere_maps(poses, W, H, FOCAL, R)
    trunc = default_trunc(LO, HI, reso)
    return fuse.tsdf_fuse(depth, opacity, poses.numpy(), FOCAL, FOCAL, W / 2, H / 2, LO, HI, reso, trunc, 0.5), trunc


def test_sphere_fuses_into_one_closed_sphere():
    tsdf, trunc = sphere_tsdf()
    assert tsdf.dtype == np.float32 and tsdf.shape == RESO
    assert np.isfinite(tsdf).all() and np.abs(tsdf).max() <= 1.0
    v, t = recon.marching_cubes(-tsdf, 0.0)
    assert len(t) > 2000
    assert recon.is_closed_oriented(t)
    assert recon.euler_characteristic(v, t) == 2
    assert recon.components(t) == 1
    p = index_to_world(v, LO, HI, RESO)
    h = (HI[0] - LO[0]) / (RESO[0] - 1)
    err = np.abs(np.linalg.norm(p, axis=1) - R)
    print(f"max | |p| - r | = {err.max():.4f} (voxel {h:.4f})")
    assert err.max() <= h
    assert recon.signed_volume(p, t) > 0                   # counter-clockwise seen from outside
    # the interior deeper than trunc is occluded from every view: inside
    x = recon.grid_points(LO, HI, RESO).astype(np.float64)
    rho = np.linalg.norm(x, axis=1)
    assert (tsdf.reshape(-1)[rho < R - trunc - 0.05] == -1.0).all()
    assert (tsdf.reshape(-1)[rho > R + 0.05] > 0).all()


def _camera(z, up):
    """A camera at (0, 0, z) looking along -z (up) or +z (not up), as a camera-to-world pose."""
    P = np.eye(4, dtype=np.float32)
    if not up:
        P[1, 1] = P[2, 2] = -1.0
    P[2, 3] = z
    return P


def test_classification_cases():
    # one camera at z = 3 looking down at an opaque plane z = 0 (depth along each pixel's unit ray), 9 x 9 pixels
    Wc = Hc = 9
    f, cx, cy = 4.0, 4.0, 4.0
    ys, xs = np.mgrid[0:Hc, 0:Wc].astype(np.float64)
    dz = 1.0 / np.sqrt(((xs - cx) / f) ** 2 + ((ys - cy) / f) ** 2 + 1.0)
    plane = (3.0 / dz).astype(np.float32)[None]
    ones, zeros = np.ones_like(plane), np.zeros_like(plane)
    lo, hi, reso = (-1.0, -1.0, -1.5), (1.0, 1.0, 1.5), (3, 3, 7)        # z = -1.5 .. 1.5 in steps of 0.5
    trunc = 0.3
    down = _camera(3.0, True)[None]
    t = fuse.tsdf_fuse(plane, ones, down, f, f, cx, cy, lo, hi, reso, trunc, 0.5)
    col = t[1, 1]                                            # the voxels on the optical axis
    assert np.array_equal(col, np.float32([-1, -1, -1, 0, 1, 1, 1]))   # occluded below, the plane at 0, free above
    # a voxel behind the camera or outside the image is seen by no view: outside
    far = fuse.tsdf_fuse(plane, ones, down, f, f, cx, cy, (-1.0, -1.0, 4.0), (1.0, 1.0, 5.0), (3, 3, 2), trunc, 0.5)
    assert (far == 1.0).all()
    wide = fuse.tsdf_fuse(plane, ones, down, f, f, cx, cy, (-50.0, 0.0, -1.0), (50.0, 0.0, -1.0), (2, 1, 1), trunc,
                          0.5)
    assert (wide == 1.0).all()
    # background pixels carve: a second camera below, looking up, sees nothing, so the occluded voxels become outside
    up = _camera(-3.0, False)[None]
    both = fuse.tsdf_fuse(np.concatenate([plane, zeros]), np.concatenate([ones, zeros]), np.concatenate([down, up]),
                          f, f, cx, cy, lo, hi, reso, trunc, 0.5)
    assert np.array_equal(both[1, 1], np.float32([1, 1, 1, 0.5, 1, 1, 1]))
    # opacity below min_opacity is background; at min_opacity it is a surface at depth / opacity
    half = np.full_like(plane, 0.5)
    assert (fuse.tsdf_fuse(plane * 0.5, half, down, f, f, cx, cy, lo, hi, reso, trunc, 0.5001) >= 1.0).all()
    assert np.array_equal(fuse.tsdf_fuse(plane * 0.5, half, down, f, f, cx, cy, lo, hi, reso, trunc, 0.5), t)


def test_off_centre_non_square_views():
    """A non-square image with an off-centre principal point still gives the sphere (the projection inverts
    util.gen_rays with its own c).  The box is tighter: these narrower views see the corners of [-1, 1]^3 only behind
    the sphere, and a voxel seen but never observed is inside."""
    poses = views(12, 3.0)
    Wn, Hn, c = 120, 80, torch.tensor([70.0, 35.0])
    depth, opacity = sphere_maps(poses, Wn, Hn, 150.0, R, c=c)
    lo, hi, reso = (-0.75,) * 3, (0.75,) * 3, (40, 40, 40)
    tsdf = fuse.tsdf_fuse(depth, opacity, poses.numpy(), 150.0, 150.0, 70.0, 35.0, lo, hi, reso,
                          default_trunc(lo, hi, reso), 0.5)
    v, t = recon.marching_cubes(-tsdf, 0.0)
    assert recon.is_closed_oriented(t) and recon.components(t) == 1
    assert recon.euler_characteristic(v, t) == 2
    h = (hi[0] - lo[0]) / (reso[0] - 1)
    assert np.abs(np.linalg.norm(index_to_world(v, lo, hi, reso), axis=1) - R).max() <= h
