"""
ORACLE -- numpy restatement of pnr_paint_vertices (csrc/pnr_recon.cu, include/pnr.h): vertex colours from rendered
views, in the kernel's float64 operation order, so that the kernel is compared against it bit for bit.

  paint_vertices  xyz, normals [n][3] float64 (world-space vertices, unit outward normals), rgb [V][H][W][3], depth,
                  opacity [V][H][W] fp32, camera-to-world poses [V][4][4] fp32, intrinsics (rounded to fp32, as the C
                  ABI takes them), trunc, min_opacity, background -> (rgb [n][3] fp32, weight [n] float64).
                  Per view: the pixel as pnr_tsdf_fuse finds it (q = R^T (x - t); q_z >= 0 or outside the image: skip).
                  Opacity a < min_opacity (or NaN): skip.  s = (depth / a - |q|) / trunc; |s| > 1 (or NaN): skip.
                  cos = n . (t - x) / |q|; cos <= 0 (or NaN): skip.  c = (rgb - background (1 - a)) / a clamped to
                  [0, 1] (NaN -> 0).  rgb = sum(cos c) / sum(cos) over the views in order, NaN with no view;
                  weight = sum(cos), 0 with no view.
"""
import numpy as np


def paint_vertices(xyz, normals, rgb, depth, opacity, poses, fx, fy, cx, cy, trunc, min_opacity, background):
    xyz = np.asarray(xyz, dtype=np.float64).reshape(-1, 3)
    normals = np.asarray(normals, dtype=np.float64).reshape(-1, 3)
    rgb = np.asarray(rgb, dtype=np.float32)
    depth = np.asarray(depth, dtype=np.float32)
    opacity = np.asarray(opacity, dtype=np.float32)
    poses = np.asarray(poses, dtype=np.float32).astype(np.float64)
    V, H, W = depth.shape
    fx, fy, cx, cy = (float(np.float32(v)) for v in (fx, fy, cx, cy))
    trunc, min_opacity, background = float(trunc), float(min_opacity), float(background)
    N = len(xyz)
    sum_c = np.zeros((N, 3))
    sum_w = np.zeros(N)
    for v in range(V):
        P = poses[v]
        d = xyz - P[:3, 3]
        q = [(P[0, j] * d[:, 0] + P[1, j] * d[:, 1]) + P[2, j] * d[:, 2] for j in range(3)]
        with np.errstate(invalid="ignore", divide="ignore", over="ignore"):
            px = cx + (fx * q[0]) / -q[2]
            py = cy + (fy * q[1]) / q[2]
            rx, ry = np.floor(px + 0.5), np.floor(py + 0.5)
            sees = (q[2] < 0) & (rx >= 0) & (rx <= W - 1) & (ry >= 0) & (ry <= H - 1)
        i = np.nonzero(sees)[0]
        iy, ix = ry[i].astype(np.int64), rx[i].astype(np.int64)
        a = opacity[v, iy, ix].astype(np.float64)
        keep = a >= min_opacity                                     # background (or NaN): no surface colour
        i, iy, ix, a = i[keep], iy[keep], ix[keep], a[keep]
        dist = np.sqrt((q[0][i] * q[0][i] + q[1][i] * q[1][i]) + q[2][i] * q[2][i])
        with np.errstate(invalid="ignore", divide="ignore", over="ignore"):
            s = (depth[v, iy, ix].astype(np.float64) / a - dist) / trunc
            keep = (s >= -1.0) & (s <= 1.0)                         # occluded or elsewhere (or NaN)
        i, iy, ix, a, dist = i[keep], iy[keep], ix[keep], a[keep], dist[keep]
        e = P[:3, 3] - xyz[i]
        nrm = normals[i]
        with np.errstate(invalid="ignore", divide="ignore", over="ignore"):
            cos = ((nrm[:, 0] * e[:, 0] + nrm[:, 1] * e[:, 1]) + nrm[:, 2] * e[:, 2]) / dist
            keep = cos > 0.0                                        # the back of the surface (or NaN)
        i, iy, ix, a, cos = i[keep], iy[keep], ix[keep], a[keep], cos[keep]
        bg = background * (1.0 - a)
        with np.errstate(invalid="ignore", divide="ignore", over="ignore"):
            c = (rgb[v, iy, ix].astype(np.float64) - bg[:, None]) / a[:, None]
            c = np.where(c > 0.0, c, 0.0)
            c = np.where(c > 1.0, 1.0, c)
        sum_c[i] += cos[:, None] * c
        sum_w[i] += cos
    painted = sum_w > 0.0
    with np.errstate(invalid="ignore", divide="ignore"):
        out = np.where(painted[:, None], sum_c / np.where(painted, sum_w, 1.0)[:, None], np.nan)
    return out.astype(np.float32), sum_w
