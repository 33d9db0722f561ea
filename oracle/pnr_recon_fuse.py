"""
ORACLE -- numpy restatement of pnr_tsdf_fuse (csrc/pnr_recon.cu, include/pnr.h): TSDF fusion of rendered depth maps,
in the kernel's float64 operation order, so that the kernel is compared against it bit for bit.

  tsdf_fuse  depth, opacity [V][H][W] fp32, camera-to-world poses [V][4][4] fp32, intrinsics (rounded to fp32, as the
             C ABI takes them), lo, hi, reso, trunc, min_opacity -> tsdf [nx][ny][nz] fp32, positive outside.
             Voxel x = pnr_grid_points' point.  Per view: q = R^T (x - t); q_z >= 0: not seen.  px = cx + fx q_x / (-q_z),
             py = cy + fy q_y / q_z, pixel = floor(p + 0.5) (ties round up); outside the image: not seen.  Opacity a of
             the pixel < min_opacity (or NaN): background, s = +1.  Else s = (depth / a - |q|) / trunc; s < -1 (or NaN):
             occluded, no observation; else min(s, 1).  tsdf = mean of the observations' s, summed in view order; with
             none, -1 when some view saw the voxel (in front of it and inside its image), else +1.
"""
import importlib.util
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_spec = importlib.util.spec_from_file_location("pnr_recon_oracle_fuse_base", os.path.join(_HERE, "pnr_recon.py"))
_recon = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(_recon)


def tsdf_fuse(depth, opacity, poses, fx, fy, cx, cy, lo, hi, reso, trunc, min_opacity):
    depth = np.asarray(depth, dtype=np.float32)
    opacity = np.asarray(opacity, dtype=np.float32)
    poses = np.asarray(poses, dtype=np.float32).astype(np.float64)
    V, H, W = depth.shape
    fx, fy, cx, cy = (float(np.float32(v)) for v in (fx, fy, cx, cy))
    trunc, min_opacity = float(trunc), float(min_opacity)
    x = _recon.grid_points(lo, hi, reso).astype(np.float64)
    N = len(x)
    total = np.zeros(N)
    count = np.zeros(N, dtype=np.int64)
    seen = np.zeros(N, dtype=bool)
    for v in range(V):
        P = poses[v]
        d = x - P[:3, 3]
        q = [(P[0, j] * d[:, 0] + P[1, j] * d[:, 1]) + P[2, j] * d[:, 2] for j in range(3)]
        with np.errstate(invalid="ignore", divide="ignore", over="ignore"):
            px = cx + (fx * q[0]) / -q[2]
            py = cy + (fy * q[1]) / q[2]
            rx, ry = np.floor(px + 0.5), np.floor(py + 0.5)
            sees = (q[2] < 0) & (rx >= 0) & (rx <= W - 1) & (ry >= 0) & (ry <= H - 1)
        seen |= sees
        i = np.nonzero(sees)[0]
        iy, ix = ry[i].astype(np.int64), rx[i].astype(np.int64)
        a = opacity[v, iy, ix].astype(np.float64)
        dep = depth[v, iy, ix].astype(np.float64)
        dist = np.sqrt((q[0][i] * q[0][i] + q[1][i] * q[1][i]) + q[2][i] * q[2][i])
        surface = a >= min_opacity
        with np.errstate(invalid="ignore", divide="ignore", over="ignore"):
            s = np.where(surface, (dep / np.where(surface, a, 1.0) - dist) / trunc, 1.0)
            obs = ~surface | (s >= -1.0)
            s = np.where(s > 1.0, 1.0, s)
        total[i[obs]] += s[obs]
        count[i[obs]] += 1
    with np.errstate(invalid="ignore", divide="ignore"):
        out = np.where(count > 0, total / np.maximum(count, 1), np.where(seen, -1.0, 1.0))
    return out.astype(np.float32).reshape(tuple(int(r) for r in reso))
