"""The vertex-painting rule (oracle/pnr_recon_paint.py, the restatement pnr_paint_vertices is compared against) on
analytic scenes: a sphere with a colour gradient, rendered from a turntable plus a top and a bottom view, fused and
meshed by the oracles, paints every vertex close to the true colour there; two solid spheres that hide each other in
some views paint every vertex with its own sphere's colour; and a semi-transparent surface composited over white paints
its colour after the background is un-mixed."""
import numpy as np

from fuse_util import views
from paint_util import fused_surface, gradient_colour, paint, sphere_scene_maps

LO, HI, RESO = (-1.0, -1.0, -1.0), (1.0, 1.0, 1.0), (48, 48, 48)
W = H = 96
FOCAL = 160.0
R = 0.5
DIST = 3.0
H_VOX = (HI[0] - LO[0]) / (RESO[0] - 1)
TRUNC = 3.0 * np.sqrt(3.0) * H_VOX                       # fuse_views' default: 3 voxel diagonals


def paint_maps(x, normals, rgb, depth, opacity, poses, trunc=TRUNC, min_opacity=0.5, background=1.0):
    return paint.paint_vertices(x, normals, rgb, depth, opacity, poses, FOCAL, FOCAL, W / 2, H / 2, trunc, min_opacity,
                                background)


def test_gradient_sphere_paints_its_colour():
    poses = views(16, DIST).numpy()
    colour = gradient_colour(R)
    rgb, depth, opacity = sphere_scene_maps(poses, W, H, FOCAL, [((0.0, 0.0, 0.0), R, colour)])
    x, t, normals = fused_surface(depth, opacity, poses, FOCAL, W / 2, H / 2, LO, HI, RESO, TRUNC)
    assert len(x) > 2000
    col, weight = paint_maps(x, normals, rgb, depth, opacity, poses)
    assert col.dtype == np.float32 and col.shape == x.shape and weight.dtype == np.float64
    assert (weight > 0).all()                              # every vertex painted
    assert np.isfinite(col).all() and col.min() >= 0.0 and col.max() <= 1.0
    # c is linear with slope 0.5 / r per channel, so the error is at most 0.5 / r times how far the painted surface
    # points lie from the vertex: the vertex's own offset from the sphere (within a voxel, as the fusion test shows),
    # plus the rounding to a pixel centre and its stretch across an oblique surface (two pixel footprints at the
    # farthest visible point, DIST / FOCAL each).
    err = np.abs(col - colour(x)).max(1)
    bound = 0.5 / R * (H_VOX + 2.0 * DIST / FOCAL)
    print(f"max colour error {err.max():.4f}, mean {err.mean():.4f}, bound {bound:.4f}")
    assert err.max() <= bound                              # observed: max 0.041, mean 0.007 (bound 0.080)
    assert err.mean() <= 0.01


A = ((-0.45, 0.0, 0.0), 0.3, (0.9, 0.2, 0.1))
B = ((0.45, 0.0, 0.0), 0.3, (0.1, 0.3, 0.8))


def two_spheres():
    """Two solid spheres on the x axis; the turntable's views along x see one in front of the other."""
    poses = views(16, DIST, phi=-10.0).numpy()
    rgb, depth, opacity = sphere_scene_maps(poses, W, H, FOCAL, [A, B])
    x, t, normals = fused_surface(depth, opacity, poses, FOCAL, W / 2, H / 2, LO, HI, RESO, TRUNC)
    near_a = np.linalg.norm(x - A[0], axis=1) < np.linalg.norm(x - B[0], axis=1)
    want = np.where(near_a[:, None], np.float32(A[2]), np.float32(B[2]))
    return poses, rgb, depth, opacity, x, normals, want


def test_occluded_views_do_not_leak():
    poses, rgb, depth, opacity, x, normals, want = two_spheres()
    col, weight = paint_maps(x, normals, rgb, depth, opacity, poses)
    painted = weight > 0
    print(f"painted {painted.sum()} of {len(x)} vertices")
    assert painted.mean() > 0.7
    assert np.abs(col[painted] - want[painted]).max() <= 1e-6
    assert np.isnan(col[~painted]).all() and (weight[~painted] == 0).all()
    # the scene does hide one sphere behind the other: accept every depth (a huge trunc) and the front sphere's
    # colour leaks onto the one behind it
    leaky, _ = paint_maps(x, normals, rgb, depth, opacity, poses, trunc=10.0)
    assert np.abs(leaky[painted] - want[painted]).max() > 0.1


def test_background_is_unmixed():
    """Opacity 0.8 with rgb = a c + (1 - a) (over white) or a c (over black), depth = a t: the painted colour is c."""
    poses, rgb, depth, opacity, x, normals, want = two_spheres()
    ref, ref_w = paint_maps(x, normals, rgb, depth, opacity, poses)
    a = np.float32(0.8)
    hit = opacity > 0
    depth8 = np.where(hit, depth * a, 0).astype(np.float32)
    op8 = np.where(hit, a, 0).astype(np.float32)
    for background in (1.0, 0.0):
        c = np.where(hit[..., None], rgb, 0.0)
        rgb8 = np.where(hit[..., None], a * c + background * (1 - a), background).astype(np.float32)
        col, weight = paint_maps(x, normals, rgb8, depth8, op8, poses, background=background)
        assert np.array_equal(weight > 0, ref_w > 0)
        painted = weight > 0
        assert np.abs(col[painted] - want[painted]).max() <= 1e-6
        assert np.abs(col[painted] - ref[painted]).max() <= 1e-6
    # below min_opacity the same pixels are background and paint nothing
    col, weight = paint_maps(x, normals, rgb, depth8, op8, poses, min_opacity=0.81)
    assert (weight == 0).all() and np.isnan(col).all()

