"""Numpy restatement of the fixed-order arithmetic of deterministic mode (csrc/pnr_determ.cu).

* `scatter_fixed`: one field-backward chunk's latent gradient in 64-bit fixed point.  The terms are the fp32 products
  d_lat * w_tap; m = max |term source| over the finite d_lat entries; e = 62 - ceil(log2(4 rows)) - E with
  m = f 2^E, f in [0.5, 1); each finite term is rounded half-to-even to an integer at scale 2^e and summed exactly in
  int64; the sum converts as float32(float64(acc) * 2^-e) and is added (fp32) into the map.  A non-finite term makes
  its element NaN.  The rounding error is at most 2^-e / 2 per term, i.e. m 2^(ceil log2(4 rows) - 63).
* `upsample_ac_backward`: the adjoint of F.interpolate(..., mode="bilinear", align_corners=True) with torch's source
  indices and lambdas, summed per input pixel in output order (oh, ow), then tap order (h-tap major), in fp32.
"""
import numpy as np


def bwd_taps(poses, focal, c, NS, Hl, Wl, C, scale, image, sb, v, x):
    """The four bilinear taps of point x (3 float32) in view v of object sb as the field backward computes them
    (csrc/pnr_geom.cuh bwd_taps, fp32, one rounding per operation, in the kernel's order) -> list of
    (channels-last offset of channel 0, float32 weight) for the taps inside the map.  poses [V][12] (world -> camera
    [3][4]), focal [n][2], c [n][2] float32; scale = latent_scaling (x, y), image = image size (w, h)."""
    f32 = np.float32
    M = poses[sb * NS + v]
    x = [f32(t) for t in x]
    q = [f32(f32(f32(M[i * 4] * x[0]) + f32(M[i * 4 + 1] * x[1])) + f32(M[i * 4 + 2] * x[2])) for i in range(3)]
    p = [f32(q[i] + M[i * 4 + 3]) for i in range(3)]
    fo = focal[sb if len(focal) > 1 else 0]
    cc = c[sb if len(c) > 1 else 0]
    u = f32(f32(f32(-p[0] / p[2]) * fo[0]) + cc[0])
    w = f32(f32(f32(-p[1] / p[2]) * fo[1]) + cc[1])
    kx, ky = f32(f32(scale[0]) / f32(image[0])), f32(f32(scale[1]) / f32(image[1]))

    def coord(t, k, n):
        i = f32(f32(f32(f32(f32(t * k) - f32(1)) + f32(1)) * f32(0.5)) * f32(n - 1))
        return f32(np.fmin(f32(n - 1), np.fmax(i, f32(0))))   # fmaxf / fminf: NaN -> 0

    ix, iy = coord(u, kx, Wl), coord(w, ky, Hl)
    x0f, y0f = f32(np.floor(ix)), f32(np.floor(iy))
    x0, y0 = int(x0f), int(y0f)
    vx1, vy1 = x0 + 1 <= Wl - 1, y0 + 1 <= Hl - 1
    x1, y1 = (x0 + 1 if vx1 else x0), (y0 + 1 if vy1 else y0)
    wx0, wx1 = f32(f32(x0f + f32(1)) - ix), f32(ix - x0f)
    wy0, wy1 = f32(f32(y0f + f32(1)) - iy), f32(iy - y0f)
    base = (sb * NS + v) * Hl * Wl * C
    off = lambda yy, xx: base + (yy * Wl + xx) * C  # noqa: E731
    taps = [(off(y0, x0), f32(wx0 * wy0))]
    if vx1:
        taps.append((off(y0, x1), f32(wx1 * wy0)))
    if vy1:
        taps.append((off(y1, x0), f32(wx0 * wy1)))
    if vx1 and vy1:
        taps.append((off(y1, x1), f32(wx1 * wy1)))
    return taps


def fixed_exponent(m, rows):
    """Scale exponent of a chunk of `rows` rows whose finite |d_lat| <= m (m float32)."""
    log2_nmax = (4 * rows - 1).bit_length()            # ceil(log2(4 rows))
    _, E = np.frexp(np.float32(m))
    return 62 - log2_nmax - int(E)


def scatter_fixed(d_latent, d_lat, taps, rows):
    """d_latent: float32 array (flat view modified in place); d_lat: float32 [rows][C] chunk rows; taps: list of
    (row, flat_offset_of_channel_0, weight float32) of the chunk, in any order -> d_latent."""
    d_lat = np.asarray(d_lat, dtype=np.float32)
    fin = np.isfinite(d_lat)
    m = np.float32(np.abs(d_lat[fin]).max()) if fin.any() else np.float32(0)
    e = fixed_exponent(m, rows)
    C = d_lat.shape[1]
    acc = np.zeros(d_latent.size, dtype=np.int64)
    nan = np.zeros(d_latent.size, dtype=bool)
    flat = d_latent.reshape(-1)
    for row, off, w in taps:
        term = d_lat[row] * np.float32(w)                        # fp32 product
        ok = np.isfinite(term)
        q = np.rint(term.astype(np.float64) * np.ldexp(1.0, e))   # exact scaling, round half to even
        idx = off + np.arange(C)
        acc[idx[ok]] += q[ok].astype(np.int64)
        nan[idx[~ok]] = True
    flat[nan] = np.float32(np.nan)
    nz = acc != 0
    flat[nz] = flat[nz] + (acc[nz].astype(np.float64) * np.ldexp(1.0, -e)).astype(np.float32)
    return d_latent


def _axis(n_in, n_out):
    scale = np.float32(n_in - 1) / np.float32(n_out - 1) if n_out > 1 else np.float32(0)
    r = (scale * np.arange(n_out, dtype=np.float32)).astype(np.float32)
    i0 = r.astype(np.int64)
    step = (i0 < n_in - 1).astype(np.int64)
    l1 = (r - i0.astype(np.float32)).astype(np.float32)
    l0 = (np.float32(1) - l1).astype(np.float32)
    return i0, step, l0, l1


def upsample_ac_backward(d_out, h_in, w_in):
    """d_out float32 [N][C][h_out][w_out] -> d_in float32 [N][C][h_in][w_in]."""
    d_out = np.asarray(d_out, dtype=np.float32)
    N, C, h_out, w_out = d_out.shape
    if (h_in, w_in) == (h_out, w_out):
        return d_out.copy()
    d_in = np.zeros((N, C, h_in, w_in), dtype=np.float32)
    hy, hs, hl0, hl1 = _axis(h_in, h_out)
    wx, ws, wl0, wl1 = _axis(w_in, w_out)
    for oh in range(h_out):
        for ow in range(w_out):
            g = d_out[:, :, oh, ow]
            for a, hl in ((0, hl0[oh]), (1, hl1[oh])):
                for b, wl in ((0, wl0[ow]), (1, wl1[ow])):
                    h, w = hy[oh] + a * hs[oh], wx[ow] + b * ws[ow]
                    d_in[:, :, h, w] = d_in[:, :, h, w] + (np.float32(hl * wl) * g).astype(np.float32)
    return d_in
