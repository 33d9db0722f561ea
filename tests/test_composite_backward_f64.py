"""`pnr_composite_backward` (k_composite_bwd, the compositing backward every training step runs once per pass) against
float64 autograd of the reference's compositing forward, on rays with near-opaque samples: the regime of a trained
pixelNeRF with hard surfaces, where a suffix sum formed by subtraction and divided by a transmittance factor of
1e-4 .. 1e-10 loses every bit.  The CUDA sources run on the host emulator (tests/cuda_emu) unmarked and on the GPU
marked `gpu`.

The bound is per ray and per output (d_field's rgb part, its sigma part, d_z):

    max_k |kernel - f64| <= C * max_k |torch_fp32 - f64| + EPS * max_k |f64|

where torch_fp32 is autograd of the same forward in float32, i.e. what the reference itself computes.  A bare relative
bound cannot work: where alpha rounds to 1 (sigma * delta >~ 17) the fp32 forward itself departs from float64 (on a ray
whose whole d_sigma is ~1e-9, torch fp32 is off by tens of percent), and so is any fp32 kernel.  A global scale would
hide a wrong ray next to a steep one.  EPS covers rays where torch fp32 happens to land close to float64: for
1 - exp(-x) at the background's small x, even correctly rounded fp32 keeps ~1e-5 relative, and the GPU's expf (2 ulp)
puts the kernel a few times further off than torch's.  With C = 16 and EPS = 5e-5 the kernel's error reaches 0.10 of
the bound on the host emulator and 0.39 on an H100 80GB HBM3 at 700 W (d_z, K = 512); a kernel that formed the suffix
sums as (total - prefix) / t exceeds it on 48 of the 56 parameter sets, by up to 5e4 (d_sigma, K = 64, surface at
sigma * delta = 100).  Where
alpha has not rounded to 1 (sigma * delta <= 15) the kernel's worst per-ray d_z and d_sigma errors, relative to the
ray's own largest value, are those of torch fp32 to two digits (<= 7.2e-3 and 2.6e-2 at sigma * delta = 15, <= 5e-5
at sigma * delta <= 8); the subtracting kernel's reached 7.5 and 2.0.
"""
import numpy as np
import pytest
import torch

import emu_util as eu

C_BOUND, EPS = 16.0, 5e-5
KS = [1, 2, 3, 64, 96, 144, 512]
PEAKS = [0.5, 2.0, 5.0, 8.0, 10.0, 12.0, 15.0, 17.0, 20.0, 25.0, 40.0, 100.0]     # sigma * delta of the surface
UPSTREAM = ["rgb", "depth", "weights", "all"]
NEAR, FAR = 0.8, 1.8


def _ray(rng, K, kind, peak=0.0, pos=0):
    """-> (z [K], sigma [K], far) in float32.  Stratified depths with jitter (the coarse sampler's layout), a
    semi-transparent background with a quarter of the sigmas <= 0, and on top of it:
      surface: sample `pos` at sigma * delta = peak;   two: surfaces at sigma * delta 8 and 12;
      clear: every sigma <= 0;   dup: the surface sample repeated (zero-length intervals, as clamped depth-centred
      samples give) with the density on the last copy;   far: the last samples clamped to far (z_last == far)."""
    z = (NEAR + (np.arange(K) + rng.uniform(0.05, 0.95, K)) / K * (FAR - NEAR)).astype(np.float32)
    sig = np.abs(rng.normal(0.0, 2.0, K)).astype(np.float32)
    sig[rng.uniform(size=K) < 0.25] = -np.abs(rng.normal(0.0, 1.0)) if K > 1 else 0.0
    far = np.float32(FAR)

    def put(k, p):
        delta = (z[k + 1] if k + 1 < K else far) - z[k]
        if delta > 0:
            sig[k] = np.float32(p / delta)

    if kind == "surface":
        put(pos, peak)
    elif kind == "two":
        put(K // 4, 8.0)
        put(min(K // 2 + 1, K - 1), 12.0)
    elif kind == "clear":
        sig[:] = -np.abs(rng.normal(0.0, 1.0, K)).astype(np.float32)
        sig[::3] = 0.0
    elif kind == "dup":
        j = K // 3
        n = min(4, K - j - 1)
        z[j:j + n + 1] = z[j]
        sig[j:j + n] = 50.0
        put(j + n, peak)
    elif kind == "far":
        n = max(1, K // 8)
        z[K - n:] = far
        sig[K - n:] = 30.0
        put(max(K - n - 1, 0), peak)
    return z, sig, far


def _batch(K, seed):
    """All the ray kinds at one K -> rays (R,8), z (R,K), field (R,K,4) float32 and one label per ray."""
    rng = np.random.default_rng(seed)
    rays = []
    for peak in PEAKS:
        for pos in sorted({0, K // 2, K - 1}):
            rays.append((f"surface sigma*delta={peak} at k={pos}", _ray(rng, K, "surface", peak, pos)))
    rays.append(("two surfaces", _ray(rng, K, "two")))
    rays.append(("transparent", _ray(rng, K, "clear")))
    for peak in (5.0, 12.0, 40.0):
        if K >= 3:
            rays.append((f"zero-length intervals, sigma*delta={peak}", _ray(rng, K, "dup", peak)))
        rays.append((f"z_last == far, sigma*delta={peak}", _ray(rng, K, "far", peak)))
    R = len(rays)
    r = torch.zeros(R, 8)
    r[:, 3:6] = torch.nn.functional.normalize(torch.from_numpy(rng.normal(size=(R, 3)).astype(np.float32)), dim=-1)
    r[:, 6] = NEAR
    r[:, 7] = torch.tensor([float(f) for _, (_, _, f) in rays])
    z = torch.from_numpy(np.stack([zz for _, (zz, _, _) in rays])).contiguous()
    sig = torch.from_numpy(np.stack([s for _, (_, s, _) in rays]))
    rgb = torch.from_numpy(rng.uniform(0.0, 1.0, (R, K, 3)).astype(np.float32))
    field = torch.cat([rgb, sig[..., None]], -1).contiguous()
    return r, z, field, [lab for lab, _ in rays]


def _upstream(which, R, K, seed):
    g = torch.Generator().manual_seed(seed)
    d_rgb, d_depth, d_w = torch.randn(R, 3, generator=g), torch.randn(R, generator=g), torch.randn(R, K, generator=g)
    return (d_rgb if which in ("rgb", "all") else None, d_depth if which in ("depth", "all") else None,
            d_w if which in ("weights", "all") else None)


def _reference(rays, z, field, white, d_rgb, d_depth, d_w, dtype):
    """Autograd of the reference's compositing (src/render/nerf.py:178-249) in `dtype` at the given float32 inputs:
    deltas with far - z_last, 1 - exp(-delta relu(sigma)), cumprod of 1 - alpha + 1e-10, weights, rgb (+ the white
    background) and depth; loss = d_rgb . rgb + d_depth depth + d_weights . weights.  -> (d_field, d_z)."""
    z = z.to(dtype).requires_grad_(True)
    field = field.to(dtype).requires_grad_(True)
    far = rays[:, -1:].to(dtype)
    deltas = torch.cat([z[:, 1:] - z[:, :-1], far - z[:, -1:]], -1)
    alphas = 1 - torch.exp(-deltas * torch.relu(field[..., 3]))
    T = torch.cumprod(torch.cat([torch.ones_like(alphas[:, :1]), 1 - alphas + 1e-10], -1), -1)
    weights = alphas * T[:, :-1]
    rgb = torch.sum(weights.unsqueeze(-1) * field[..., :3], -2)
    depth = torch.sum(weights * z, -1)
    if white:
        rgb = rgb + 1 - weights.sum(dim=1).unsqueeze(-1)
    loss = torch.zeros((), dtype=dtype)
    for out, up in ((rgb, d_rgb), (depth, d_depth), (weights, d_w)):
        if up is not None:
            loss = loss + (out * up.to(dtype)).sum()
    return torch.autograd.grad(loss, [field, z])


def _parts(d_field, d_z):
    return {"d_field rgb": d_field[..., :3].reshape(d_z.shape[0], -1), "d_sigma": d_field[..., 3], "d_z": d_z}


def _per_ray_ratio(got, ref64, ref32):
    """-> {part: (R,) error over bound} for got / float32 reference against the float64 reference."""
    out = {}
    g, r64, r32 = _parts(*got), _parts(*ref64), _parts(*ref32)
    for k in g:
        err = (g[k].double() - r64[k]).abs().amax(-1)
        bound = C_BOUND * (r32[k].double() - r64[k]).abs().amax(-1) + EPS * r64[k].abs().amax(-1)
        out[k] = torch.where(err == 0, torch.zeros_like(err), err / bound)
    return out


def check(call, K, white, which):
    """call(rays, z, field, white, d_rgb, d_depth, d_w) -> (d_field, d_z) on the CPU.  Asserts the per-ray bound."""
    seed = 1000 * K + 10 * white + UPSTREAM.index(which)
    rays, z, field, labels = _batch(K, seed)
    R = rays.shape[0]
    d_rgb, d_depth, d_w = _upstream(which, R, K, seed)
    got = call(rays, z, field, white, d_rgb, d_depth, d_w)
    ref64 = _reference(rays, z, field, white, d_rgb, d_depth, d_w, torch.float64)
    ref32 = _reference(rays, z, field, white, d_rgb, d_depth, d_w, torch.float32)
    assert ref64[0].abs().max() > 0
    assert torch.isfinite(got[0]).all() and torch.isfinite(got[1]).all()
    assert torch.all(got[0][..., 3][field[..., 3] <= 0] == 0)        # no density gradient where sigma <= 0
    if d_rgb is None:
        assert torch.all(got[0][..., :3] == 0)
    ratios = _per_ray_ratio(got, ref64, ref32)
    for part, rr in ratios.items():
        i = int(torch.argmax(rr))
        assert rr[i] <= 1.0, (part, labels[i], f"error {rr[i].item():.3g} x the bound")
    return ratios, labels


def _emulated(rays, z, field, white, d_rgb, d_depth, d_w):
    R, K = z.shape
    d_field, d_z = torch.full((R, K, 4), float("nan")), torch.full((R, K), float("nan"))
    eu.ok(eu.lib().pnr_composite_backward(eu.ptr(rays), eu.ptr(z), eu.ptr(field), white, eu.ptr(d_rgb),
                                          eu.ptr(d_depth), eu.ptr(d_w), eu.ptr(d_field), eu.ptr(d_z), R, K, None))
    return d_field, d_z


def _on_gpu(rays, z, field, white, d_rgb, d_depth, d_w):
    import gpu_util  # noqa: F401  (puts the package on sys.path)
    import pnr_native as pn
    dev = torch.device("cuda:0")
    R, K = z.shape
    cu = lambda t: t.to(dev).contiguous() if t is not None else None
    a = [cu(t) for t in (rays, z, field, d_rgb, d_depth, d_w)]
    d_field = torch.full((R, K, 4), float("nan"), device=dev)
    d_z = torch.full((R, K), float("nan"), device=dev)
    pn.check(pn.lib().pnr_composite_backward(pn.dptr(a[0]), pn.dptr(a[1]), pn.dptr(a[2]), white, pn.dptr(a[3]),
                                             pn.dptr(a[4]), pn.dptr(a[5]), pn.dptr(d_field), pn.dptr(d_z), R, K,
                                             pn.stream_ptr(dev)))
    torch.cuda.synchronize(dev)
    return d_field.cpu(), d_z.cpu()


@pytest.mark.parametrize("which", UPSTREAM)
@pytest.mark.parametrize("white", [0, 1])
@pytest.mark.parametrize("K", KS)
def test_emulated_composite_backward_within_fp32_of_float64(K, white, which):
    check(_emulated, K, white, which)


@pytest.mark.gpu
@pytest.mark.parametrize("which", UPSTREAM)
@pytest.mark.parametrize("white", [0, 1])
@pytest.mark.parametrize("K", KS)
def test_gpu_composite_backward_within_fp32_of_float64(K, white, which):
    check(_on_gpu, K, white, which)


def test_the_cases_reach_opacity():
    """The surface sweep spans alpha well short of 1 to alpha rounded to 1 in float32, and the float64 d_sigma at the
    surface is not negligible on the rays where cancellation used to bite."""
    rays, z, field, labels = _batch(64, 0)
    far = rays[:, -1:]
    deltas = torch.cat([z[:, 1:] - z[:, :-1], far - z[:, -1:]], -1)
    sd = deltas * torch.relu(field[..., 3])
    alpha32 = 1 - torch.exp(-sd)
    assert (alpha32 < 0.5).any() and (alpha32 == 1).any()
    assert ((sd > 7.5) & (sd < 16.5) & (alpha32 < 1)).sum() >= 9
    assert any("zero-length" in lab for lab in labels) and any("z_last" in lab for lab in labels)
    assert (deltas == 0).any(-1).sum() >= 6
