"""Per-ray check of a render's fine pass, with no budget of excused rays -- test infrastructure.

The importance samples are a deterministic function of the kernel's own coarse weights and the noise, and the fine
outputs a deterministic function of the merged samples, so every ray can be checked against a reference that is
conditioned on the kernel's own coarse pass:

  1. `check_fused_equals_stage`: the fused render's merged samples are bit-equal to the stage kernel `pnr_sample_fine`
     run on the render's own z_coarse / weights_coarse / depth_coarse with the same noise.  Both run
     `sample_fine_ray` (csrc/pnr_ray_ops.cuh) one warp per ray with explicit round-to-nearest intrinsics, so any
     difference is a bug.  Needs the CUDA library.
  2. `explain_fine_z`: the merged samples against a float64 inverse cdf built from the same fp32 coarse weights.  Each
     importance sample must be the fp32 sample of a bin its `u` admits (a bin other than the float64 one only when `u`
     lies within fp32 rounding of the cdf edge between them), the depth-centred samples must be bit-equal to their fp32
     formula, nothing else may be in the merge, and the merge must be sorted.
  3. `check_fine_outputs`: the fine rgb / depth / weights against the oracle's compositing of the field at the
     kernel's own merged samples, on every ray (or a fixed subset of a large render).

Row order everywhere is the renderer's: row = sb * B + b.
"""
from collections import Counter

import numpy as np
import torch

import golden_util as gu

U32 = 2.0 ** -24          # unit roundoff of fp32


def cdf_eps(Kc):
    """Bound on |cdf32[k] - cdf64[k]| for the kernel's fp32 cdf (csrc/pnr_ray_ops.cuh sample_fine_ray).

    The kernel forms t_i = fl(w_i + 1e-5f), the total T = fl(sum t_i) by per-lane sums and a shuffle tree, p_i =
    fl(t_i / T) and cdf32[k] = fl(cdf32[k-1] + p_{k-1}) sequentially.  With u = 2^-24 and all terms positive, to first
    order:
      * t_i: one rounding, plus the constant 1e-5f differing from 1e-5 by < 1e-5 u       -> 2 u relative,
      * T: any summation order of Kc positive terms errs by at most (Kc - 1) u relative  -> (Kc - 1) u,
      * p_i: one rounding                                                                 -> 1 u,
      * cdf32[k]: k - 1 <= Kc - 1 sequential additions of positive terms                 -> (Kc - 1) u relative,
    so |cdf32[k] - cdf64[k]| <= (2 Kc + 1) u * cdf64[k] <= (2 Kc + 1) u since cdf64 <= 1.  One more u covers the
    second-order terms: eps = (2 Kc + 4) u."""
    return (2 * Kc + 4) * U32


def _np32(t):
    if isinstance(t, torch.Tensor):
        return t.detach().cpu().float().numpy()
    return np.asarray(t, dtype=np.float32)


def stage_fine_z(rays, z_coarse, w_coarse, d_coarse, noise, Kc, Kf, Kfd, depth_std):
    """pnr_sample_fine (the stage kernel) on cuda:0 -> merged samples (R, Kc + Kf) on the device."""
    import pnr_native as pn
    dev = torch.device("cuda:0")
    d = lambda t: None if t is None else t.detach().to(dev, torch.float32).contiguous()
    r8 = d(rays.reshape(-1, 8))
    R, Ku = r8.shape[0], Kf - Kfd
    zc, wc, dc = d(z_coarse.reshape(R, Kc)), d(w_coarse.reshape(R, Kc)), d(d_coarse.reshape(R))
    u = d(noise["u_fine"]) if Ku > 0 else None
    uj = d(noise["u_fine_jit"]) if Ku > 0 else None
    nd = d(noise["n_depth"]) if Kfd > 0 else None
    zf = torch.empty(R, Kc + Kf, device=dev)
    L = pn.lib()
    pn.check(L.pnr_sample_fine(pn.dptr(r8), pn.dptr(zc), pn.dptr(wc), pn.dptr(dc), pn.dptr(u), pn.dptr(uj),
                               pn.dptr(nd), float(depth_std), pn.dptr(zf), R, Kc, Kf, Kfd, pn.stream_ptr(dev)))
    torch.cuda.synchronize(dev)
    return zf


def check_fused_equals_stage(rays, coarse, z_fine, noise, Kc, Kf, Kfd, depth_std):
    """Layer 1.  coarse: dict(z, weights, depth) of the fused render; z_fine its merged samples (R, Kc + Kf)."""
    ref = stage_fine_z(rays, coarse["z"], coarse["weights"], coarse["depth"], noise, Kc, Kf, Kfd, depth_std)
    got = z_fine.detach().to(ref.device).reshape(ref.shape)
    if not torch.equal(got, ref):
        bad = (got != ref).any(-1).nonzero().flatten().tolist()
        raise AssertionError(f"fused merge differs from pnr_sample_fine on {len(bad)} rays, first {bad[:8]}")


def explain_fine_z(rays, z_coarse, w_coarse, d_coarse, noise, Kc, Kf, Kfd, depth_std, z_fine):
    """Layer 2.  Raises AssertionError naming the first ray whose merged samples are not explained; returns the number
    of importance samples that took an admissible bin other than the float64 cdf's."""
    r8 = _np32(rays).reshape(-1, 8)
    R, K, Ku = r8.shape[0], Kc + Kf, Kf - Kfd
    near, far = r8[:, 6:7], r8[:, 7:8]
    zc, zf = _np32(z_coarse).reshape(R, Kc), _np32(z_fine).reshape(R, K)
    unsorted = ~(zf[:, 1:] >= zf[:, :-1]).all(-1)
    if unsorted.any():
        raise AssertionError(f"ray {int(np.argmax(unsorted))}: merged samples are not sorted")
    fixed = [zc]
    if Kfd > 0:
        dc = _np32(d_coarse).reshape(R, 1)
        nd = _np32(noise["n_depth"]).reshape(R, Kfd)
        fixed.append(np.maximum(np.minimum(dc + nd * np.float32(depth_std), far), near))
    fixed = np.concatenate(fixed, axis=1)
    if Ku == 0:
        bad = ~(np.sort(fixed, axis=1) == zf).all(-1)
        if bad.any():
            r = int(np.argmax(bad))
            _multiset_rest(zf[r], fixed[r], r)          # names the missing sample
            raise AssertionError(f"ray {r}: merged samples hold values that are no sample")
        return 0
    w = _np32(w_coarse).reshape(R, Kc).astype(np.float64) + 1e-5
    cdf = np.concatenate([np.zeros((R, 1)), np.cumsum(w / w.sum(-1, keepdims=True), axis=1)], axis=1)   # (R, Kc+1)
    u = _np32(noise["u_fine"]).reshape(R, Ku)
    uj = _np32(noise["u_fine_jit"]).reshape(R, Ku)
    u64 = u.astype(np.float64)[:, :, None]
    eps = cdf_eps(Kc)
    # bin i in [0, Kc] holds u when cdf[i] <= u < cdf[i + 1] (bin Kc: u past the last edge)
    lo = cdf[:, None, :]
    hi = np.concatenate([cdf[:, 1:], np.full((R, 1), np.inf)], axis=1)[:, None, :]
    primary = np.maximum((lo <= u64).sum(-1) - 1, 0)                                   # (R, Ku)
    admissible = (lo - eps <= u64) & (u64 < hi + eps)                                 # (R, Ku, Kc+1)
    # the fp32 sample of every bin: s = (i + u_jit) / Kc, z = near (1 - s) + far s
    s = (np.arange(Kc + 1, dtype=np.float32)[None, None, :] + uj[:, :, None]) / np.float32(Kc)
    cand = near[:, :, None] * (np.float32(1.0) - s) + far[:, :, None] * s            # (R, Ku, Kc+1) fp32
    zp = np.take_along_axis(cand, primary[:, :, None], axis=2)[:, :, 0]
    exact = (np.sort(np.concatenate([fixed, zp], axis=1), axis=1) == zf).all(-1)
    moved = 0
    for r in np.nonzero(~exact)[0].tolist():
        moved += _assign(_multiset_rest(zf[r], fixed[r], r), cand[r], admissible[r], primary[r], r)
    return moved


def _multiset_rest(merged, fixed, r):
    """merged minus the multiset `fixed` (coarse and depth-centred samples), as a list; raises when one is missing."""
    rest = Counter(merged.tolist())
    for v in fixed.tolist():
        if rest[v] == 0:
            raise AssertionError(f"ray {r}: the coarse or depth-centred sample {v!r} is missing from the merge")
        rest[v] -= 1
    return [v for v, n in rest.items() for _ in range(n)]


def _assign(rest, cand, admissible, primary, r):
    """Matches the remaining merged values one-to-one to importance samples, each to the sample of an admissible bin,
    preferring the float64 bin; returns how many took another bin."""
    from scipy.optimize import linear_sum_assignment
    Ku = cand.shape[0]
    if len(rest) != Ku:
        raise AssertionError(f"ray {r}: {len(rest)} merged values remain for {Ku} importance samples")
    big = 1e9
    cost = np.full((Ku, Ku), big)
    val = np.asarray(rest, dtype=np.float32)
    for j in range(Ku):
        ok = admissible[j]
        for m in range(Ku):
            hit = ok & (cand[j] == val[m])
            if hit[primary[j]]:
                cost[j, m] = 0.0
            elif hit.any():
                cost[j, m] = 1.0
    rows, cols = linear_sum_assignment(cost)
    if (cost[rows, cols] >= big).any():
        j = int(rows[np.argmax(cost[rows, cols])])
        raise AssertionError(f"ray {r}: importance sample {j} is not the sample of any bin its u admits "
                             f"(admissible bins {np.nonzero(admissible[j])[0].tolist()}, merged rest {sorted(rest)})")
    return int(cost[rows, cols].sum())


def oracle_composite(state, latent, w, NS, white_bkgd, eval_batch_size=50000, arithmetic=None):
    """composite(rays (n, 8), z (n, K), sb) -> (weights, rgb, depth) of the oracle's field at z.  `arithmetic`: an
    optional context manager factory that swaps the field's arithmetic (tests/tc_fast_oracle.py)."""
    def composite(rays, z, sb):
        with torch.no_grad():
            if arithmetic is None:
                return gu.oracle.composite(rays, z, sb, state, latent, w, NS, white_bkgd, eval_batch_size)
            with arithmetic():
                return gu.oracle.composite(rays, z, sb, state, latent, w, NS, white_bkgd, eval_batch_size)
    return composite


def case_composite(case, fine=True, arithmetic=None):
    """oracle_composite for a golden case's scene: the fine MLP (the coarse one when mlp_fine is None) or the coarse."""
    cfg = case["cfg"]
    w = case["wf"] if (fine and case["wf"] is not None) else case["wc"]
    return oracle_composite(gu.oracle_state(case), case["latent"], w, cfg["NS"], bool(cfg["white_bkgd"]),
                            cfg["eval_batch_size"], arithmetic)


def subset_rows(SB, B, n, seed=0):
    """A fixed random subset of about n rays, the same columns of every object -> (columns, rows)."""
    per = max(1, min(B, n // SB))
    cols = torch.randperm(B, generator=torch.Generator().manual_seed(seed))[:per].sort().values
    rows = (torch.arange(SB)[:, None] * B + cols[None, :]).reshape(-1)
    return cols, rows


def check_fine_outputs(rays, z, out, composite, rgb_tol=1e-4, depth_tol=1e-4, weights_tol=1e-4, n_sub=None,
                       what="fine"):
    """Layer 3.  rays (SB, B, 8); z (SB*B, K) the kernel's samples; out: dict(rgb (SB*B, 3), depth (SB*B,), optional
    weights (SB*B, K)) of the kernel at z.  Compares against composite(...) on every ray, or on a fixed subset of
    n_sub rays.  A tolerance of None skips that output.  Returns the max |d| per output.  `what` names the pass in
    messages (the same check serves the coarse pass at the coarse samples)."""
    SB, B = rays.shape[0], rays.shape[1]
    r = rays.detach().cpu().float()
    rows = torch.arange(SB * B)
    if n_sub is not None and n_sub < SB * B:
        cols, rows = subset_rows(SB, B, n_sub)
        r = r[:, cols]
    zz = z.detach().cpu().float().reshape(SB * B, -1)[rows].contiguous()
    w_ref, rgb_ref, dep_ref = composite(r.reshape(-1, 8).contiguous(), zz, SB)
    errs = {}
    for key, ref, tol in (("rgb", rgb_ref, rgb_tol), ("depth", dep_ref, depth_tol), ("weights", w_ref, weights_tol)):
        if tol is None or out.get(key) is None:
            continue
        got = out[key].detach().cpu().float().reshape(SB * B, -1)[rows]
        d = (got - ref.reshape(got.shape)).abs().amax(-1)
        errs[key] = float(d.max())
        if not bool((d < tol).all()):       # NaN fails too
            bad = (~(d < tol)).nonzero().flatten()
            raise AssertionError(f"{what} {key} of {bad.numel()} rays (first: row {int(rows[bad[0]])}) differs from "
                                 f"the reference at the kernel's samples: max {errs[key]:.3e} >= {tol:.0e}")
    return errs


def check_render(rays, coarse, fine, noise, Kc, Kf, Kfd, depth_std, composite, stage=True, n_sub=None, **tols):
    """Layers 1 (when `stage`), 2 and 3 of a render's fine pass.  rays (SB, B, 8); coarse / fine: dicts of the render's
    z, weights, depth (and fine rgb).  Returns dict(moved=<importance samples in a non-float64 bin>, **max errors)."""
    if stage:
        check_fused_equals_stage(rays, coarse, fine["z"], noise, Kc, Kf, Kfd, depth_std)
    moved = explain_fine_z(rays, coarse["z"], coarse["weights"], coarse["depth"], noise, Kc, Kf, Kfd, depth_std,
                           fine["z"])
    errs = check_fine_outputs(rays, fine["z"], fine, composite, n_sub=n_sub, **tols)
    return dict(moved=moved, **errs)


def simt_composite(net, white_bkgd):
    """composite(...) for layer 3 on the GPU: the fine field of `net` on the fp32 SIMT engine at the given samples,
    composited by pnr_composite.  For renders too large for the CPU oracle."""
    import pnr_native as pn

    def composite(rays, z, sb):
        dev = torch.device("cuda:0")
        r, zz = rays.to(dev).contiguous(), z.to(dev).contiguous()
        R, K = zz.shape
        pts = (r[:, None, :3] + zz[..., None] * r[:, None, 3:6]).reshape(sb, -1, 3)
        dirs = r[:, None, 3:6].expand(-1, K, -1).reshape(sb, -1, 3)
        engine = net.engine
        net.engine = "simt"
        try:
            with torch.no_grad():
                field = net(pts, coarse=False, viewdirs=dirs).reshape(R, K, 4).contiguous()
        finally:
            net.engine = engine
        w, rgb, dep = torch.empty(R, K, device=dev), torch.empty(R, 3, device=dev), torch.empty(R, device=dev)
        pn.check(pn.lib().pnr_composite(pn.dptr(r), pn.dptr(zz), pn.dptr(field), 1 if white_bkgd else 0, pn.dptr(w),
                                        pn.dptr(rgb), pn.dptr(dep), R, K, pn.stream_ptr(dev)))
        torch.cuda.synchronize(dev)
        return w.cpu(), rgb.cpu(), dep.cpu()
    return composite


def check_true_shape(bench, net, renderer, cfg, rays_dev, n=256, arithmetic=None, n_sub=None, **tols):
    """Layers 1-3 on the rays and noise of bench.parity_block (n rays spread over the frame, noise seed 7), rendered
    again with weights; layer 3 against the oracle on the scene bench.build_scene made."""
    R = rays_dev.shape[1]
    idx = torch.linspace(0, R - 1, min(n, R)).long()
    sub = rays_dev[:, idx.to(rays_dev.device)].contiguous()
    Kc, Kf, Kfd = cfg["n_coarse"], cfg["n_fine"], cfg["n_fine_depth"]
    noise = bench.synth.draw_noise(7, sub.shape[1], Kc, Kf, Kfd)
    with torch.no_grad():
        out = renderer._forward_fused(net, sub, want_weights=True,
                                      noise_in={k: v.to(sub.device) for k, v in noise.items()}, want_z=True)
    src, _, focal, c = bench.synth.make_cameras(cfg)
    state = gu.oracle.encode_state(src, focal, c[None], cfg["W"], cfg["H"])
    w = {k: v.detach().float().cpu() for k, v in net.mlp_fine.state_dict().items()}
    comp = oracle_composite(state, net.encoder.latent.detach().float().cpu(), w, cfg["NS"], cfg["white_bkgd"],
                            arithmetic=arithmetic)
    pick = lambda o: dict(z=o.z, weights=o.weights, depth=o.depth, rgb=o.rgb)
    return check_render(sub, pick(out.coarse), pick(out.fine), noise, Kc, Kf, Kfd, renderer.depth_std, comp,
                        n_sub=n_sub, **tols)


def check_case(case, res, depth_std=0.01, stage=True, arithmetic=None, **tols):
    """check_render for a golden-style case (tests/golden_util.py) and its render `res` (tests/gpu_util.py
    render_case_cuda: dict(coarse=..., fine=...) with want_weights and want_z)."""
    cfg = case["cfg"]
    return check_render(case["rays"], res["coarse"], res["fine"], case["noise"], cfg["n_coarse"], cfg["n_fine"],
                        cfg["n_fine_depth"], depth_std, case_composite(case, arithmetic=arithmetic), stage=stage,
                        **tols)
