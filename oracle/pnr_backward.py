"""
ORACLE -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

Hand-derived backward pass of the training loss (SURVEY.md 8f-1): the gradient formulas a fused
backward kernel has to implement, written stage by stage in plain torch WITHOUT autograd, so that
each formula can be checked on the CPU before any CUDA exists.  `tests/test_oracle_backward.py`
checks this module against (a) autograd through `pnr_oracle.train_loss` and (b) the gradients the
reference itself produced (`tests/golden/grad_*.npz`, `oracle/make_golden.py::grad_fixture`).

What carries gradient in the reference (src/render/nerf.py:251-303, train/train.py:199-215):
  * both passes' MLP weights and the latent, through field values -> compositing -> MSE;
  * sample depths: points = o + z d (nerf.py:185) feed pos-enc, projection and the bilinear
    gather, and deltas/depth depend on z (nerf.py:178-182, 240).  z_coarse and the inverse-CDF
    samples carry no parameter gradient (the coarse weights are detached, nerf.py:286), but the
    depth-centred samples do: z = clamp(depth_coarse + N*std) with depth_coarse NOT detached
    (nerf.py:289-291), so the fine loss reaches the coarse MLP through d(depth_coarse).
"""
import importlib.util
import math
import os

import torch
import torch.nn.functional as F

_HERE = os.path.dirname(os.path.abspath(__file__))
_spec = importlib.util.spec_from_file_location("pnr_oracle", os.path.join(_HERE, "pnr_oracle.py"))
oracle = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(oracle)


def _mm(a, b):
    """Every GEMM of the backward goes through here (scripts/precision_study_backward.py swaps in reduced-precision
    emulations to size the tensor-core version)."""
    return a @ b


def _linear(x, w, b):
    """Every layer of field_forward_saved goes through here (tests/test_gpu_backward_wide.py swaps in the split-bf16
    operands of the CUDA backward's recomputed forward)."""
    return F.linear(x, w, b)


# ----------------------------------------------------------------------------------------
# compositing (nerf.py:178-182, 222-249)
# ----------------------------------------------------------------------------------------
def exclusive_suffix(x):
    """sum_{m>k} x_m along the last axis, summed from the back.  Not (inclusive sum - x_k): behind a near-opaque sample
    both terms are that sample's g w and their difference, later divided by t_k ~ 1e-4 .. 1e-10, is all rounding."""
    rev = torch.flip(torch.cumsum(torch.flip(x, [-1]), -1), [-1])
    return torch.cat([rev[..., 1:], torch.zeros_like(rev[..., :1])], -1)


def composite_backward(rays, z, field, d_rgb, d_depth, white_bkgd):
    """field (B,K,4) = (rgb_k, sigma_k) as PixelNeRFNet.forward returns them; d_rgb (B,3), d_depth (B,).
    Forward: delta_k = z_{k+1} - z_k (last: far - z_{K-1}); s_k = relu(sigma_k); e_k = exp(-delta_k s_k);
    a_k = 1 - e_k; t_k = e_k + 1e-10; T_k = prod_{j<k} t_j; w_k = a_k T_k; rgb = sum w_k c_k (+ 1 - sum w_k);
    depth = sum w_k z_k.  Returns d_field (B,K,4), d_z (B,K)."""
    B, K = z.shape
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
    d_a = g_w * T - exclusive_suffix(g_w * w) / t
    d_s = d_a * e * deltas
    d_delta = d_a * e * s
    d_field = torch.empty_like(field)
    d_field[..., :3] = w.unsqueeze(-1) * d_rgb.unsqueeze(1)
    d_field[..., 3] = d_s * (sig > 0).float()
    d_z = w * d_depth.unsqueeze(1) - d_delta
    d_z[:, 1:] += d_delta[:, :-1]
    return d_field, d_z


# ----------------------------------------------------------------------------------------
# field (models.py:146-266, resnetfc.py:132-184, encoder.py:80-109, code.py:30-42)
# ----------------------------------------------------------------------------------------
def _posenc_tables(num_freqs=6, freq_factor=1.5):
    freqs = freq_factor * 2.0 ** torch.arange(0, num_freqs)
    f = torch.repeat_interleave(freqs, 2)            # (12,)
    ph = torch.zeros(2 * num_freqs)
    ph[1::2] = math.pi * 0.5
    return f, ph


def field_forward_saved(xyz, viewdirs, state, latent, w, NS, n_blocks=5, combine_layer=3):
    """Same arithmetic as pnr_oracle.field_eval, keeping what the backward needs."""
    SB, P, _ = xyz.shape
    V, C, Hl, Wl = latent.shape
    poses = state["poses"]
    R = poses[:, :3, :3]                                                    # (V,3,3)
    x = xyz.unsqueeze(1).expand(-1, NS, -1, -1).reshape(SB * NS, P, 3)
    x_rot = torch.matmul(R[:, None], x.unsqueeze(-1))[..., 0]
    x_cam = x_rot + poses[:, None, :3, 3]
    zf, lat, uv = oracle.field_inputs(xyz, viewdirs, state, latent, NS)
    sv = dict(SB=SB, P=P, NS=NS, R=R, x_rot=x_rot.reshape(-1, 3), x_cam=x_cam, uv=uv, feat=zf, lat=lat,
              latent_shape=latent.shape, n_blocks=n_blocks, combine_layer=combine_layer, w=w, state=state,
              latent=latent, blocks=[])
    h = _linear(zf, w["lin_in.weight"], w["lin_in.bias"])
    for b in range(n_blocks):
        if b == combine_layer and NS > 1:
            h = h.reshape(-1, NS, P, h.shape[-1]).mean(dim=1).reshape(-1, h.shape[-1])
        if b < combine_layer:
            h = h + _linear(lat, w[f"lin_z.{b}.weight"], w[f"lin_z.{b}.bias"])
        a = torch.relu(h)
        n = _linear(a, w[f"blocks.{b}.fc_0.weight"], w[f"blocks.{b}.fc_0.bias"])
        r = torch.relu(n)
        sv["blocks"].append(dict(h_pre=h, a=a, n=n, r=r))
        h = h + _linear(r, w[f"blocks.{b}.fc_1.weight"], w[f"blocks.{b}.fc_1.bias"])
    sv["h_last"] = h
    o4 = _linear(torch.relu(h), w["lin_out.weight"], w["lin_out.bias"]).reshape(SB, P, 4)
    sv["o4"] = o4
    out = torch.cat((torch.sigmoid(o4[..., :3]), torch.relu(o4[..., 3:4])), dim=-1)
    return out, sv


def gather_backward(sv, d_lat):
    """Backward of encoder.index (encoder.py:80-109): d_lat (rows,C) -> (d_latent (V,C,Hl,Wl), d_uv (V,P,2))."""
    V, C, Hl, Wl = sv["latent_shape"]
    latent, uv, image_shape = sv["latent"], sv["uv"], sv["state"]["image_shape"]
    P = uv.shape[1]
    scale = oracle.latent_scaling(latent) / image_shape
    g = uv * scale - 1.0
    ix_u = ((g[..., 0] + 1.0) / 2.0) * (Wl - 1)
    iy_u = ((g[..., 1] + 1.0) / 2.0) * (Hl - 1)
    ix = torch.clamp(ix_u, 0.0, float(Wl - 1))
    iy = torch.clamp(iy_u, 0.0, float(Hl - 1))
    x0, y0 = torch.floor(ix), torch.floor(iy)
    x1, y1 = x0 + 1.0, y0 + 1.0
    lat_hw = latent.permute(0, 2, 3, 1)
    vidx = torch.arange(V).view(V, 1).expand(V, P)
    dl = d_lat.reshape(V, P, C)
    d_latent_hw = torch.zeros(V, Hl, Wl, C)
    d_ix = torch.zeros(V, P)
    d_iy = torch.zeros(V, P)
    # tap (xx, yy) has weight wx(xx) * wy(yy); d weight / d ix = +-wy, d weight / d iy = +-wx
    for xx, wx, sx in ((x0, x1 - ix, -1.0), (x1, ix - x0, 1.0)):
        for yy, wy, sy in ((y0, y1 - iy, -1.0), (y1, iy - y0, 1.0)):
            inb = ((xx >= 0) & (xx <= Wl - 1) & (yy >= 0) & (yy <= Hl - 1)).float()
            xi, yi = xx.clamp(0, Wl - 1).long(), yy.clamp(0, Hl - 1).long()
            d_latent_hw.index_put_((vidx, yi, xi), dl * (wx * wy * inb).unsqueeze(-1), accumulate=True)
            dot = (dl * lat_hw[vidx, yi, xi]).sum(-1) * inb
            d_ix += dot * sx * wy
            d_iy += dot * sy * wx
    # clamp passes the gradient inside [0, size-1] (inclusive, like torch.clamp)
    d_ix = d_ix * ((ix_u >= 0) & (ix_u <= Wl - 1)).float()
    d_iy = d_iy * ((iy_u >= 0) & (iy_u <= Hl - 1)).float()
    d_uv = torch.stack((d_ix * scale[0] * 0.5 * (Wl - 1), d_iy * scale[1] * 0.5 * (Hl - 1)), dim=-1)
    return d_latent_hw.permute(0, 3, 1, 2), d_uv


def field_backward(sv, d_out):
    """d_out (SB,P,4) w.r.t. (sigmoid rgb, relu sigma) -> (grads {name: tensor}, d_latent, d_xyz (SB,P,3))."""
    SB, P, NS, w = sv["SB"], sv["P"], sv["NS"], sv["w"]
    nb, cl = sv["n_blocks"], sv["combine_layer"]
    o4 = sv["o4"]
    rgb = torch.sigmoid(o4[..., :3])
    d_o4 = torch.cat((d_out[..., :3] * rgb * (1 - rgb), d_out[..., 3:4] * (o4[..., 3:4] > 0).float()), -1).reshape(-1, 4)
    g = {}
    h_last = sv["h_last"]
    g["lin_out.weight"] = _mm(d_o4.t(), torch.relu(h_last))
    g["lin_out.bias"] = d_o4.sum(0)
    d_h = _mm(d_o4, w["lin_out.weight"]) * (h_last > 0).float()
    d_lat = torch.zeros_like(sv["lat"])
    for b in range(nb - 1, -1, -1):
        s = sv["blocks"][b]
        g[f"blocks.{b}.fc_1.weight"] = _mm(d_h.t(), s["r"])
        g[f"blocks.{b}.fc_1.bias"] = d_h.sum(0)
        d_n = _mm(d_h, w[f"blocks.{b}.fc_1.weight"]) * (s["n"] > 0).float()
        g[f"blocks.{b}.fc_0.weight"] = _mm(d_n.t(), s["a"])
        g[f"blocks.{b}.fc_0.bias"] = d_n.sum(0)
        d_h = d_h + _mm(d_n, w[f"blocks.{b}.fc_0.weight"]) * (s["h_pre"] > 0).float()
        if b < cl:
            g[f"lin_z.{b}.weight"] = _mm(d_h.t(), sv["lat"])
            g[f"lin_z.{b}.bias"] = d_h.sum(0)
            d_lat = d_lat + _mm(d_h, w[f"lin_z.{b}.weight"])
        if b == cl and NS > 1:                           # mean over views (util.py:461-471)
            d = d_h.shape[-1]
            d_h = (d_h.reshape(SB, 1, P, d) / NS).expand(-1, NS, -1, -1).reshape(-1, d)
    g["lin_in.weight"] = _mm(d_h.t(), sv["feat"])
    g["lin_in.bias"] = d_h.sum(0)
    d_feat = _mm(d_h, w["lin_in.weight"])                    # (rows, 42)
    # positional encoding (code.py:30-42): channels [x(3), sin(x f_k + ph_k) for k in 0..11 (3 each)], then 3 view dirs
    f, ph = _posenc_tables()
    xr = sv["x_rot"]
    d_xrot = d_feat[:, :3].clone()
    enc = d_feat[:, 3:39].reshape(-1, 12, 3)
    d_xrot += (enc * torch.cos(xr.unsqueeze(1) * f.view(1, -1, 1) + ph.view(1, -1, 1)) * f.view(1, -1, 1)).sum(1)
    # gather and projection (encoder.py:80-109, models.py:206-212)
    d_latent, d_uv = gather_backward(sv, d_lat)
    focal, c = sv["state"]["focal"], sv["state"]["c"]
    fo = focal.unsqueeze(1)
    fo = fo.unsqueeze(1).expand(-1, NS, -1, -1).reshape(-1, 1, 2) if focal.shape[0] > 1 else fo
    xc = sv["x_cam"]
    gz = d_uv * fo                                        # d(-xy/z)
    d_xcam = torch.empty_like(xc)
    d_xcam[..., :2] = -gz / xc[..., 2:]
    d_xcam[..., 2] = (gz * xc[..., :2]).sum(-1) / (xc[..., 2] * xc[..., 2])
    d_xr = d_xrot.reshape(SB * NS, P, 3) + d_xcam
    d_x = torch.matmul(sv["R"][:, None].transpose(-1, -2), d_xr.unsqueeze(-1))[..., 0]     # R^T d
    d_xyz = d_x.reshape(SB, NS, P, 3).sum(1)
    return g, d_latent, d_xyz


# ----------------------------------------------------------------------------------------
# whole training loss (train/train.py:199-215 over nerf.py:251-303)
# ----------------------------------------------------------------------------------------
def _pass_forward(rays, z, sb, state, latent, w, NS):
    B, K = z.shape
    points = (rays[:, None, :3] + z.unsqueeze(2) * rays[:, None, 3:6]).reshape(sb, -1, 3)
    viewdirs = rays[:, None, 3:6].expand(-1, K, -1).reshape(sb, -1, 3)
    out, sv = field_forward_saved(points, viewdirs, state, latent, w, NS)
    return out.reshape(B, K, 4), sv


def _pass_backward(rays, z, sv, field, d_rgb, d_depth, white_bkgd):
    d_field, d_z = composite_backward(rays, z, field, d_rgb, d_depth, white_bkgd)
    g, d_latent, d_xyz = field_backward(sv, d_field.reshape(sv["SB"], -1, 4))
    d_z = d_z + (d_xyz.reshape(z.shape[0], z.shape[1], 3) * rays[:, None, 3:6]).sum(-1)     # points = o + z d
    return g, d_latent, d_z


def train_loss_backward(rays, rgb_gt, noise, state, latent, w_coarse, w_fine, NS, n_coarse, n_fine, n_fine_depth,
                        depth_std=0.01, white_bkgd=True, lambda_coarse=1.0, lambda_fine=1.0):
    """-> (loss, grads_coarse, grads_fine_or_None, d_latent) of pnr_oracle.train_loss, no autograd."""
    with torch.no_grad():
        sb = rays.shape[0]
        rays = rays.reshape(-1, 8)
        gt = rgb_gt.reshape(-1, 3)
        z_c = oracle.sample_coarse(rays, noise["u_coarse"], n_coarse)
        f_c, sv_c = _pass_forward(rays, z_c, sb, state, latent, w_coarse, NS)
        w_c, rgb_c, depth_c = oracle.composite_from_field(rays, z_c, f_c, white_bkgd)
        loss = F.mse_loss(rgb_c, gt)
        d_rgb_c = 2.0 * (rgb_c - gt) / gt.numel()
        d_depth_c = torch.zeros_like(depth_c)
        g_f = None
        d_latent = torch.zeros_like(latent)
        if n_fine > 0:
            d_rgb_c = d_rgb_c * lambda_coarse
            samps = [z_c]
            if n_fine - n_fine_depth > 0:
                samps.append(oracle.sample_fine(rays, w_c, noise["u_fine"], noise["u_fine_jit"], n_coarse))
            if n_fine_depth > 0:
                z_unclamped = depth_c.unsqueeze(1) + noise["n_depth"] * depth_std
                samps.append(oracle.sample_fine_depth(rays, depth_c, noise["n_depth"], depth_std))
            z_f, order = torch.sort(torch.cat(samps, dim=-1), dim=-1)
            wf = w_fine if w_fine is not None else w_coarse
            f_f, sv_f = _pass_forward(rays, z_f, sb, state, latent, wf, NS)
            _, rgb_f, _ = oracle.composite_from_field(rays, z_f, f_f, white_bkgd)
            loss = loss * lambda_coarse + F.mse_loss(rgb_f, gt) * lambda_fine
            d_rgb_f = 2.0 * (rgb_f - gt) / gt.numel() * lambda_fine
            g_f, dl_f, d_zf = _pass_backward(rays, z_f, sv_f, f_f, d_rgb_f, torch.zeros_like(depth_c), white_bkgd)
            d_latent += dl_f
            if n_fine_depth > 0:
                d_cat = torch.zeros_like(d_zf).scatter_(1, order, d_zf)          # undo the sort
                d_zd = d_cat[:, -n_fine_depth:]
                inside = (z_unclamped >= rays[:, -2:-1]) & (z_unclamped <= rays[:, -1:])   # clamp(nerf.py:160)
                d_depth_c = (d_zd * inside.float()).sum(-1)
        g_c, dl_c, _ = _pass_backward(rays, z_c, sv_c, f_c, d_rgb_c, d_depth_c, white_bkgd)
        d_latent += dl_c
        if n_fine > 0 and w_fine is None:                 # one MLP serves both passes
            g_c = {k: g_c[k] + g_f[k] for k in g_c}
            g_f = None
        return loss, g_c, g_f, d_latent
