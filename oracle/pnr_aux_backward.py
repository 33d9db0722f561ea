"""
ORACLE -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

Hand-derived backward of the renderer for upstream gradients of ALL SIX outputs of NeRFRenderer.forward (rgb, depth
and weights of both passes), in plain torch without autograd.  It extends `pnr_backward.py` (whose loss, train.py's
rgb MSEs, only produces rgb gradients) with the two terms a loss on depth or weights adds:
  * compositing: the per-sample weight gradient becomes g_k = d_rgb . c_k + d_depth z_k (- sum d_rgb if white)
    + d_weights_k; the rest of the compositing backward is unchanged;
  * the coarse depth: its gradient is the caller's d_depth_coarse plus the share of the depth-centred fine samples
    (nerf.py:289-291), which now also carry the fine depth / weights gradients.
`tests/test_oracle_aux_backward.py` checks this module against autograd through `pnr_oracle.render` and against the
gradients the reference produced itself (`tests/golden/grad_aux_*.npz`, `oracle/make_golden_aux.py`).
"""
import importlib.util
import os

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
_spec = importlib.util.spec_from_file_location("pnr_backward", os.path.join(_HERE, "pnr_backward.py"))
bw = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(bw)
oracle = bw.oracle

OUTPUTS = ("d_rgb_coarse", "d_depth_coarse", "d_weights_coarse", "d_rgb_fine", "d_depth_fine", "d_weights_fine")


def composite_backward(rays, z, field, d_rgb, d_depth, d_weights, white_bkgd):
    """pnr_backward.composite_backward with an upstream gradient of the weights as well: d_rgb (B,3), d_depth (B,),
    d_weights (B,K); each may be None (zero).  Returns d_field (B,K,4), d_z (B,K) (compositing's own terms only)."""
    B, K = z.shape
    d_rgb = torch.zeros(B, 3) if d_rgb is None else d_rgb
    d_depth = torch.zeros(B) if d_depth is None else d_depth
    far = rays[:, -1:]
    deltas = torch.cat([z[:, 1:] - z[:, :-1], far - z[:, -1:]], -1)
    c, sig = field[..., :3], field[..., 3]
    s = torch.relu(sig)
    e = torch.exp(-deltas * s)
    a = 1 - e
    t = e + 1e-10
    T = torch.cumprod(torch.cat([torch.ones_like(t[:, :1]), t], -1), -1)[:, :-1]
    w = a * T
    g_w = (d_rgb.unsqueeze(1) * c).sum(-1) + d_depth.unsqueeze(1) * z
    if white_bkgd:
        g_w = g_w - d_rgb.sum(-1, keepdim=True)
    if d_weights is not None:
        g_w = g_w + d_weights
    d_a = g_w * T - bw.exclusive_suffix(g_w * w) / t
    d_s = d_a * e * deltas
    d_delta = d_a * e * s
    d_field = torch.empty_like(field)
    d_field[..., :3] = w.unsqueeze(-1) * d_rgb.unsqueeze(1)
    d_field[..., 3] = d_s * (sig > 0).float()
    d_z = w * d_depth.unsqueeze(1) - d_delta
    d_z[:, 1:] += d_delta[:, :-1]
    return d_field, d_z


def _pass_backward(rays, z, sv, field, d_rgb, d_depth, d_weights, white_bkgd):
    d_field, d_z = composite_backward(rays, z, field, d_rgb, d_depth, d_weights, white_bkgd)
    g, d_latent, d_xyz = bw.field_backward(sv, d_field.reshape(sv["SB"], -1, 4))
    d_z = d_z + (d_xyz.reshape(z.shape[0], z.shape[1], 3) * rays[:, None, 3:6]).sum(-1)     # points = o + z d
    return g, d_latent, d_z


def render_backward(rays, noise, state, latent, w_coarse, w_fine, NS, n_coarse, n_fine, n_fine_depth, up,
                    depth_std=0.01, white_bkgd=True):
    """Backward of pnr_oracle.render for upstream gradients of all six outputs; generalises
    pnr_backward.train_loss_backward.  up: dict keyed by OUTPUTS with tensors of shape (R,3) / (R,) / (R,K), any key
    missing or None = zero.  -> (grads_coarse, grads_fine_or_None, d_latent)."""
    with torch.no_grad():
        sb = rays.shape[0]
        rays = rays.reshape(-1, 8)
        R = rays.shape[0]
        get = lambda k, *shape: None if up.get(k) is None else up[k].reshape(R, *shape)
        z_c = oracle.sample_coarse(rays, noise["u_coarse"], n_coarse)
        f_c, sv_c = bw._pass_forward(rays, z_c, sb, state, latent, w_coarse, NS)
        w_c, _, depth_c = oracle.composite_from_field(rays, z_c, f_c, white_bkgd)
        d_depth_c = get("d_depth_coarse")
        d_depth_c = torch.zeros(R) if d_depth_c is None else d_depth_c
        g_f = None
        d_latent = torch.zeros_like(latent)
        if n_fine > 0:
            K = n_coarse + n_fine
            samps = [z_c]
            if n_fine - n_fine_depth > 0:
                samps.append(oracle.sample_fine(rays, w_c, noise["u_fine"], noise["u_fine_jit"], n_coarse))
            if n_fine_depth > 0:
                z_unclamped = depth_c.unsqueeze(1) + noise["n_depth"] * depth_std
                samps.append(oracle.sample_fine_depth(rays, depth_c, noise["n_depth"], depth_std))
            z_f, order = torch.sort(torch.cat(samps, dim=-1), dim=-1)
            wf = w_fine if w_fine is not None else w_coarse
            f_f, sv_f = bw._pass_forward(rays, z_f, sb, state, latent, wf, NS)
            g_f, dl_f, d_zf = _pass_backward(rays, z_f, sv_f, f_f, get("d_rgb_fine", 3), get("d_depth_fine"),
                                             get("d_weights_fine", K), white_bkgd)
            d_latent += dl_f
            if n_fine_depth > 0:
                d_cat = torch.zeros_like(d_zf).scatter_(1, order, d_zf)          # undo the sort
                d_zd = d_cat[:, -n_fine_depth:]
                inside = (z_unclamped >= rays[:, -2:-1]) & (z_unclamped <= rays[:, -1:])   # clamp(nerf.py:160)
                d_depth_c = d_depth_c + (d_zd * inside.float()).sum(-1)
        g_c, dl_c, _ = _pass_backward(rays, z_c, sv_c, f_c, get("d_rgb_coarse", 3), d_depth_c,
                                      get("d_weights_coarse", n_coarse), white_bkgd)
        d_latent += dl_c
        if n_fine > 0 and w_fine is None:                 # one MLP serves both passes
            g_c = {k: g_c[k] + g_f[k] for k in g_c}
            g_f = None
        return g_c, g_f, d_latent
