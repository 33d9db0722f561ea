"""pnr_paint_vertices (csrc/pnr_recon.cu) on the host emulator (built by tests/recon_emu.py): the colours and weights
bit for bit against the numpy oracle (oracle/pnr_recon_paint.py) on random maps and on every branch of the rule --
projections on a rounding tie, vertices behind a camera and outside its image, background pixels and NaN opacity, |s|
exactly at, just inside and just outside 1, back-facing views, vertices no view paints -- with one view and with no
vertices, and the error codes."""
import ctypes as C

import numpy as np
import pytest
import torch

import emu_util as eu
import recon_emu
from paint_util import paint

PNR_ERR_INVALID = -1


def _f64(a):
    return torch.from_numpy(np.ascontiguousarray(a, dtype=np.float64))


def _f32(a):
    return torch.from_numpy(np.ascontiguousarray(a, dtype=np.float32))


def _p(t):
    return C.c_void_p(t.data_ptr())


def emu_paint(xyz, normals, rgb, depth, opacity, poses, fx, fy, cx, cy, trunc, min_opacity, background):
    n = len(xyz)
    pad = lambda a: np.concatenate([np.reshape(a, (-1, 3)), np.zeros((1, 3))])  # noqa: E731  (never NULL, n = 0 too)
    xyz, normals = _f64(pad(xyz)), _f64(pad(normals))
    rgb, depth, opacity, poses = _f32(rgb), _f32(depth), _f32(opacity), _f32(poses)
    V, H, W = depth.shape
    out = torch.full((max(n, 1), 3), 7.0)
    weight = torch.full((max(n, 1),), 7.0, dtype=torch.float64)
    rc = recon_emu.lib().pnr_paint_vertices(_p(xyz), _p(normals), n, eu.ptr(rgb), eu.ptr(depth), eu.ptr(opacity), V,
                                            W, H, eu.ptr(poses), fx, fy, cx, cy, trunc, min_opacity, background,
                                            eu.ptr(out), _p(weight), None)
    assert rc == 0, recon_emu.lib().pnr_last_error().decode()
    return out.numpy()[:n], weight.numpy()[:n]


def assert_same(*args):
    got, got_w = emu_paint(*args)
    want, want_w = paint.paint_vertices(*args)
    assert got.shape == want.shape and got_w.shape == want_w.shape
    assert np.array_equal(got.view(np.int32), want.view(np.int32))
    assert np.array_equal(got_w.view(np.int64), want_w.view(np.int64))
    return got, got_w


def random_case(seed, n=300, V=5, W=11, H=7):
    g = np.random.default_rng(seed)
    import util
    poses = torch.stack([util.pose_spherical(float(g.uniform(-180, 180)), float(g.uniform(-80, 80)),
                                             float(g.uniform(0.3, 2.0))) for _ in range(V)]).numpy()
    poses[:, :3, 3] += g.uniform(-0.3, 0.3, (V, 3)).astype(np.float32)   # some cameras inside the box
    opacity = g.choice(np.float32([0.0, 0.2, 0.4999999, 0.5, 0.5000001, 0.8, 1.0]), size=(V, H, W))
    depth = (opacity * g.uniform(0.0, 3.0, (V, H, W))).astype(np.float32)
    rgb = g.uniform(-0.2, 1.2, (V, H, W, 3)).astype(np.float32)          # some outside [0, 1]: the clamp
    rgb.flat[::97] = np.nan                                               # which takes NaN to 0
    xyz = g.uniform(-1.0, 1.0, (n, 3))
    normals = g.normal(size=(n, 3))
    normals /= np.linalg.norm(normals, axis=1, keepdims=True)
    return xyz, normals, rgb, depth, opacity, poses


@pytest.mark.parametrize("seed", range(4))
@pytest.mark.parametrize("background", [0.0, 1.0, 0.37])
def test_random_maps(seed, background):
    xyz, normals, rgb, depth, opacity, poses = random_case(seed)
    col, w = assert_same(xyz, normals, rgb, depth, opacity, poses, 6.0, 5.5, 6.3, 2.75, 0.5, 0.5, background)
    painted = w > 0
    assert painted.any() and (~painted).any()
    assert np.isnan(col[~painted]).all() and (w[~painted] == 0).all()
    assert (col[painted] >= 0).all() and (col[painted] <= 1).all()


def down_camera():
    """A camera at z = 3 looking down -z, as a camera-to-world pose [1, 4, 4]."""
    P = np.eye(4, dtype=np.float32)
    P[2, 3] = 3.0
    return P[None]


UP = (0.0, 0.0, 1.0)


def test_rounding_ties_and_visibility():
    """fx = 3 and cx = 2: vertex x of the plane z = 0 projects to 2 + x, so half-integer x land exactly on ties, which
    round up; vertices above z = 3 are behind the camera and those with |x| or |y| large outside the image.  trunc is
    large, so every pixel the vertex lands on paints it: the colour tells which pixel that was."""
    g = np.random.default_rng(5)
    W, H = 6, 5
    rgb = g.uniform(0.0, 1.0, (1, H, W, 3)).astype(np.float32)
    depth, opacity = np.full((1, H, W), 3.0, np.float32), np.ones((1, H, W), np.float32)
    s = np.arange(-3.0, 3.01, 0.5)
    X, Y = np.meshgrid(s, s, indexing="ij")
    plane = np.stack([X.ravel(), Y.ravel(), np.zeros(X.size)], 1)
    above = np.array([[0.0, 0.0, 3.0], [0.0, 0.0, 3.5], [0.5, -0.5, 4.0]])
    xyz = np.concatenate([plane, above])
    normals = np.broadcast_to(UP, xyz.shape)
    col, w = assert_same(xyz, normals, rgb, depth, opacity, down_camera(), 3.0, 3.0, 2.0, 2.0, 100.0, 0.5, 1.0)
    inside = (X.ravel() >= -2.5) & (X.ravel() < 3.5) & (Y.ravel() > -2.5) & (Y.ravel() <= 2.5)
    assert np.array_equal(w[:len(plane)] > 0, inside)
    # the tie x = 0.5 (pixel 2.5) rounds up to pixel 3; -y is up, so y = -0.5 (pixel 2.5) rounds to row 3 as well
    k = np.nonzero((plane[:, 0] == 0.5) & (plane[:, 1] == -0.5))[0][0]
    assert np.array_equal(col[k], rgb[0, 3, 3])
    assert (w[len(plane):] == 0).all() and np.isnan(col[len(plane):]).all()
    # the same through a non-square image with an off-centre principal point and unequal focals
    assert_same(xyz, normals, np.resize(rgb, (1, 9, 11, 3)), np.full((1, 9, 11), 3.0, np.float32),
                np.ones((1, 9, 11), np.float32), down_camera(), 2.0, 4.0, 1.0, 3.0, 100.0, 1.0, 0.0)


def test_background_and_nan_opacity():
    """Opacity below min_opacity or NaN skips the view; at min_opacity it paints."""
    rgb = np.full((1, 3, 3, 3), 0.25, np.float32)
    xyz, normals = np.zeros((1, 3)), np.array([UP])
    for a, painted in ((0.0, False), (0.49999997, False), (float("nan"), False), (0.5, True), (1.0, True)):
        opacity = np.full((1, 3, 3), a, np.float32)
        depth = (opacity * 3.0).astype(np.float32)
        col, w = assert_same(xyz, normals, rgb, depth, opacity, down_camera(), 3.0, 3.0, 1.0, 1.0, 0.1, 0.5, 0.0)
        assert (w[0] > 0) == painted, a


def test_truncation_bounds():
    """The vertex (0, 0, z) on the optical axis is at distance 3 - z from the camera, which sees depth 3.5 there:
    s = (3.5 - (3 - z)) / 0.5 = 1 + 2 z.  |s| = 1 paints, just past it does not."""
    rgb = np.full((1, 3, 3, 3), 0.75, np.float32)
    depth, opacity = np.full((1, 3, 3), 3.5, np.float32), np.ones((1, 3, 3), np.float32)
    eps = 1e-12
    z = np.array([0.0, -eps, eps, -0.5, -1.0, -1.0 + eps, -1.0 - eps])
    xyz = np.stack([np.zeros_like(z), np.zeros_like(z), z], 1)
    col, w = assert_same(xyz, np.broadcast_to(UP, xyz.shape), rgb, depth, opacity, down_camera(), 3.0, 3.0, 1.0, 1.0,
                         0.5, 0.5, 1.0)
    assert np.array_equal(w > 0, [True, True, False, True, True, True, False])
    assert (col[w > 0] == np.float32(0.75)).all()


def test_back_facing_views():
    """A normal away from the camera, or perpendicular to the ray (cos = 0), does not paint; a tilted one paints with
    weight cos."""
    rgb = np.full((1, 3, 3, 3), 0.5, np.float32)
    depth, opacity = np.full((1, 3, 3), 3.0, np.float32), np.ones((1, 3, 3), np.float32)
    normals = np.array([[0.0, 0.0, -1.0], [1.0, 0.0, 0.0], [0.0, 0.6, -0.8], [0.0, 0.6, 0.8], UP])
    xyz = np.zeros_like(normals)
    col, w = assert_same(xyz, normals, rgb, depth, opacity, down_camera(), 3.0, 3.0, 1.0, 1.0, 0.1, 0.5, 0.0)
    assert np.array_equal(w[[0, 1, 2, 4]], [0.0, 0.0, 0.0, 1.0]) and abs(w[3] - 0.8) < 1e-15


def test_views_in_order():
    """Several views each see the vertex: the mean is cos-weighted and summed in view order; one view alone, and a
    vertex no view paints (NaN, weight 0)."""
    import util
    poses = torch.stack([util.pose_spherical(float(a), -20.0, 2.0) for a in (-60, -20, 0, 30, 70, 180)]).numpy()
    g = np.random.default_rng(9)
    V, H, W = len(poses), 9, 9
    rgb = g.uniform(0.0, 1.0, (V, H, W, 3)).astype(np.float32)
    depth, opacity = np.full((V, H, W), 2.0, np.float32), np.ones((V, H, W), np.float32)
    xyz = np.array([[0.0, 0.0, 0.0], [0.01, -0.02, 0.03], [5.0, 5.0, 5.0]])
    up = poses[:, :3, 3].astype(np.float64).mean(0)        # towards the cameras, all above the vertex
    tilted = up + np.array([0.3, -0.2, 0.1])
    normals = np.stack([up, tilted, up]) / np.linalg.norm([up, tilted, up], axis=1, keepdims=True)
    col, w = assert_same(xyz, normals, rgb, depth, opacity, poses, 9.0, 9.0, 4.0, 4.0, 0.2, 0.5, 1.0)
    assert (w[:2] > 0).all() and w[2] == 0 and np.isnan(col[2]).all()
    col1, w1 = assert_same(xyz, normals, rgb[:1], depth[:1], opacity[:1], poses[:1], 9.0, 9.0, 4.0, 4.0, 0.2, 0.5, 1.0)
    assert (w1 <= w).all()


def test_no_vertices():
    got, got_w = emu_paint(np.zeros((0, 3)), np.zeros((0, 3)), np.zeros((1, 2, 2, 3)), np.ones((1, 2, 2)),
                           np.ones((1, 2, 2)), np.eye(4)[None], 1.0, 1.0, 0.5, 0.5, 0.1, 0.5, 1.0)
    assert got.shape == (0, 3) and got_w.shape == (0,)


def test_error_codes():
    L = recon_emu.lib()
    xyz, nrm = _f64(np.zeros((2, 3))), _f64(np.tile(UP, (2, 1)))
    rgb, depth = torch.ones(1, 3, 4, 3), torch.ones(1, 3, 4)
    poses = torch.eye(4)[None].contiguous()
    out, weight = torch.empty(2, 3), _f64(np.zeros(2))

    def call(x=_p(xyz), nr=_p(nrm), n=2, c=eu.ptr(rgb), d=eu.ptr(depth), o=eu.ptr(depth), V=1, W=4, H=3,
             p=eu.ptr(poses), trunc=0.1, m=0.5, bg=1.0, co=eu.ptr(out), w=_p(weight)):
        return L.pnr_paint_vertices(x, nr, n, c, d, o, V, W, H, p, 1.0, 1.0, 2.0, 1.5, trunc, m, bg, co, w, None)
    assert call() == 0
    assert call(n=0) == 0
    for kw in (dict(x=None), dict(nr=None), dict(c=None), dict(d=None), dict(o=None), dict(p=None), dict(co=None),
               dict(w=None), dict(n=-1), dict(V=0), dict(W=0), dict(H=-1), dict(trunc=0.0), dict(trunc=-1.0),
               dict(trunc=float("nan")), dict(trunc=float("inf")), dict(m=0.0), dict(m=1.0000001), dict(m=float("nan")),
               dict(bg=float("nan")), dict(bg=float("inf")), dict(bg=float("-inf"))):
        assert call(**kw) == PNR_ERR_INVALID, kw
    assert call(m=1.0, bg=-0.5) == 0
