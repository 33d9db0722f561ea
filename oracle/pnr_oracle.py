"""
ORACLE -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

CPU (torch fp32) restatement of pixelNeRF's volume-rendering hot path, one function per
stage with every random draw passed in explicitly.  Only `tests/`,
`__graft_entry__.smoke()` and `bench.py`'s cpu_baseline / `--impl reference` legs may
import this module; the product path (pixel-nerf_b200/) never does and fails loudly when
its CUDA library is missing.

Parity pinning: the reference ships NO tests or golden vectors for this path
(SURVEY.md section 4), so the oracle is pinned against outputs of the reference itself,
generated in the build container by `oracle/make_golden.py` (which imports
/root/reference/src unmodified) and committed under `tests/golden/*.npz`;
`tests/test_oracle_golden.py` replays them.

Each function cites the reference lines it follows (paths relative to /root/reference).
Row order everywhere is the reference's "view-major" order: row = (sb*NS + v)*P + p
(src/model/models.py:161, src/util/util.py:58-65).
"""
import math

import torch
import torch.nn.functional as F

# ----------------------------------------------------------------------------------------
# scene state: what PixelNeRFNet.encode leaves behind (src/model/models.py:89-144)
# ----------------------------------------------------------------------------------------


def encode_state(poses_c2w, focal, c, W, H):
    """poses_c2w (V,4,4); focal scalar | (V,) | (V,2); c None | scalar | (V,) | (V,2).
    Returns dict(poses (V,3,4) world->cam, focal (F,2) with fy negated, c (C,2),
    image_shape [W,H]).  models.py:112-141."""
    rot = poses_c2w[:, :3, :3].transpose(1, 2)
    trans = -torch.bmm(rot, poses_c2w[:, :3, 3:])
    poses = torch.cat((rot, trans), dim=-1)
    image_shape = torch.tensor([float(W), float(H)])
    focal = torch.as_tensor(focal, dtype=torch.float32)
    if focal.dim() == 0:
        focal = focal[None, None].repeat((1, 2))
    elif focal.dim() == 1:
        focal = focal.unsqueeze(-1).repeat((1, 2))
    else:
        focal = focal.clone()
    focal = focal.float()
    focal[..., 1] *= -1.0
    if c is None:
        c = (image_shape * 0.5).unsqueeze(0)
    else:
        c = torch.as_tensor(c, dtype=torch.float32)
        if c.dim() == 0:
            c = c[None, None].repeat((1, 2))
        elif c.dim() == 1:
            c = c.unsqueeze(-1).repeat((1, 2))
    return dict(poses=poses, focal=focal, c=c, image_shape=image_shape)


def latent_scaling(latent):
    """encoder.py:161-163: (Wl, Hl) / ((Wl, Hl) - 1) * 2."""
    s = torch.tensor([float(latent.shape[-1]), float(latent.shape[-2])])
    return s / (s - 1) * 2.0


# ----------------------------------------------------------------------------------------
# field stages (src/model/models.py:146-266)
# ----------------------------------------------------------------------------------------


def positional_encoding(x, num_freqs=6, freq_factor=1.5):
    """code.py:11-42: cat(x, sin(x*f_k + phase)), f repeated twice, phases (0, pi/2)."""
    freqs = freq_factor * 2.0 ** torch.arange(0, num_freqs)
    f = torch.repeat_interleave(freqs, 2).view(1, -1, 1)
    ph = torch.zeros(2 * num_freqs)
    ph[1::2] = math.pi * 0.5
    ph = ph.view(1, -1, 1)
    e = x.unsqueeze(1).repeat(1, num_freqs * 2, 1)
    e = torch.sin(torch.addcmul(ph, e, f))
    e = e.view(x.shape[0], -1)
    return torch.cat((x, e), dim=-1)


def bilinear_border_gather(latent, uv, image_shape):
    """encoder.py:80-109 restated without grid_sample.
    latent (V,C,Hl,Wl), uv (V,P,2) in source-image pixels -> (V,P,C).
    grid_sample(align_corners=True, padding_mode='border', bilinear): unnormalise
    ((g+1)/2*(size-1)), clip to [0,size-1], taps floor / floor+1, out-of-range taps add 0."""
    V, C, Hl, Wl = latent.shape
    scale = latent_scaling(latent) / image_shape
    g = uv * scale - 1.0
    ix = ((g[..., 0] + 1.0) / 2.0) * (Wl - 1)
    iy = ((g[..., 1] + 1.0) / 2.0) * (Hl - 1)
    ix = torch.clamp(ix, 0.0, float(Wl - 1))
    iy = torch.clamp(iy, 0.0, float(Hl - 1))
    x0 = torch.floor(ix)
    y0 = torch.floor(iy)
    x1 = x0 + 1.0
    y1 = y0 + 1.0
    w_nw = (x1 - ix) * (y1 - iy)
    w_ne = (ix - x0) * (y1 - iy)
    w_sw = (x1 - ix) * (iy - y0)
    w_se = (ix - x0) * (iy - y0)
    lat = latent.permute(0, 2, 3, 1)  # (V,Hl,Wl,C)
    vidx = torch.arange(V).view(V, 1).expand(V, uv.shape[1])

    def tap(xx, yy, w):
        inb = (xx >= 0) & (xx <= Wl - 1) & (yy >= 0) & (yy <= Hl - 1)
        xi = xx.clamp(0, Wl - 1).long()
        yi = yy.clamp(0, Hl - 1).long()
        return lat[vidx, yi, xi] * (w * inb.float()).unsqueeze(-1)

    out = tap(x0, y0, w_nw)
    out = out + tap(x1, y0, w_ne)
    out = out + tap(x0, y1, w_sw)
    out = out + tap(x1, y1, w_se)
    return out


def resnetfc(w, zx, NS, P, d_latent=512, n_blocks=5, combine_layer=3):
    """resnetfc.py:132-184 (beta=0 -> ReLU, no SPADE, combine_type average).
    w: state_dict-shaped dict; zx (rows, d_latent + d_in), rows = SB*NS*P view-major."""
    z = zx[..., :d_latent]
    x = zx[..., d_latent:]
    x = F.linear(x, w["lin_in.weight"], w["lin_in.bias"])
    for blk in range(n_blocks):
        if blk == combine_layer and not (NS == 1):
            # util.py:461-471 combine_interleaved: reshape(-1, NS, P, d).mean(1)
            x = x.reshape(-1, NS, P, x.shape[-1]).mean(dim=1).reshape(-1, x.shape[-1])
        if blk < combine_layer:
            x = x + F.linear(z, w[f"lin_z.{blk}.weight"], w[f"lin_z.{blk}.bias"])
        # resnetfc.py:53-62 ResnetBlockFC, shortcut None
        net = F.linear(torch.relu(x), w[f"blocks.{blk}.fc_0.weight"], w[f"blocks.{blk}.fc_0.bias"])
        dx = F.linear(torch.relu(net), w[f"blocks.{blk}.fc_1.weight"], w[f"blocks.{blk}.fc_1.bias"])
        x = x + dx
    return F.linear(torch.relu(x), w["lin_out.weight"], w["lin_out.bias"])


def field_inputs(xyz, viewdirs, state, latent, NS):
    """models.py:158-227: per (view, point) the 42 geometric channels and the 512 gathered
    latent channels.  xyz, viewdirs (SB,P,3).  Returns (z_feature (rows,42), latent (rows,512),
    uv (SB*NS,P,2))."""
    SB, P, _ = xyz.shape
    poses = state["poses"]
    x = xyz.unsqueeze(1).expand(-1, NS, -1, -1).reshape(SB * NS, P, 3)  # repeat_interleave
    xyz_rot = torch.matmul(poses[:, None, :3, :3], x.unsqueeze(-1))[..., 0]
    xyz_cam = xyz_rot + poses[:, None, :3, 3]
    z_feature = positional_encoding(xyz_rot.reshape(-1, 3))  # use_xyz & normalize_z (models.py:171)
    vd = viewdirs.reshape(SB, P, 3, 1)
    vd = vd.unsqueeze(1).expand(-1, NS, -1, -1, -1).reshape(SB * NS, P, 3, 1)
    vd = torch.matmul(poses[:, None, :3, :3], vd).reshape(-1, 3)
    z_feature = torch.cat((z_feature, vd), dim=1)  # models.py:188-196

    uv = -xyz_cam[:, :, :2] / xyz_cam[:, :, 2:]
    focal, c = state["focal"], state["c"]
    fo = focal.unsqueeze(1)
    fo = fo.unsqueeze(1).expand(-1, NS, -1, -1).reshape(-1, 1, 2) if focal.shape[0] > 1 else fo
    cc = c.unsqueeze(1)
    cc = cc.unsqueeze(1).expand(-1, NS, -1, -1).reshape(-1, 1, 2) if c.shape[0] > 1 else cc
    uv = uv * fo
    uv = uv + cc
    lat = bilinear_border_gather(latent, uv, state["image_shape"])  # (SB*NS,P,512)
    return z_feature, lat.reshape(-1, latent.shape[1]), uv


def field_eval(xyz, viewdirs, state, latent, w, NS):
    """PixelNeRFNet.forward (models.py:146-266) for the shipped feature set -> (SB,P,4)."""
    SB, P, _ = xyz.shape
    zf, lat, _ = field_inputs(xyz, viewdirs, state, latent, NS)
    zx = torch.cat((lat, zf), dim=-1)
    out = resnetfc(w, zx, NS, P).reshape(-1, P, 4)
    rgb = torch.sigmoid(out[..., :3])
    sigma = torch.relu(out[..., 3:4])
    return torch.cat((rgb, sigma), dim=-1).reshape(SB, P, 4)


# ----------------------------------------------------------------------------------------
# renderer stages (src/render/nerf.py)
# ----------------------------------------------------------------------------------------


def sample_coarse(rays, u, n_coarse):
    """nerf.py:98-113 (lindisp False).  rays (B,8), u (B,Kc) ~ U[0,1)."""
    near, far = rays[:, -2:-1], rays[:, -1:]
    step = 1.0 / n_coarse
    z_steps = torch.linspace(0, 1 - step, n_coarse).unsqueeze(0).repeat(rays.shape[0], 1)
    z_steps = z_steps + u * step
    return near * (1 - z_steps) + far * z_steps


def sample_fine(rays, weights, u, u_jit, n_coarse):
    """nerf.py:120-148.  weights (B,Kc), u/u_jit (B,Kf-Kfd)."""
    weights = weights + 1e-5
    pdf = weights / torch.sum(weights, -1, keepdim=True)
    cdf = torch.cumsum(pdf, -1)
    cdf = torch.cat([torch.zeros_like(cdf[:, :1]), cdf], -1)
    inds = torch.searchsorted(cdf, u, right=True).float() - 1.0
    inds = torch.clamp_min(inds, 0.0)
    z_steps = (inds + u_jit) / n_coarse
    near, far = rays[:, -2:-1], rays[:, -1:]
    return near * (1 - z_steps) + far * z_steps


def sample_fine_depth(rays, depth, n, depth_std):
    """nerf.py:150-161.  n (B,Kfd) ~ N(0,1)."""
    z = depth.unsqueeze(1).repeat((1, n.shape[1]))
    z = z + n * depth_std
    return torch.max(torch.min(z, rays[:, -1:]), rays[:, -2:-1])


def composite_from_field(rays, z_samp, out, white_bkgd):
    """nerf.py:178-182 and :222-249.  out (B,K,4) = sigmoid rgb, relu sigma."""
    deltas = z_samp[:, 1:] - z_samp[:, :-1]
    delta_inf = rays[:, -1:] - z_samp[:, -1:]
    deltas = torch.cat([deltas, delta_inf], -1)
    rgbs = out[..., :3]
    sigmas = out[..., 3]
    alphas = 1 - torch.exp(-deltas * torch.relu(sigmas))
    alphas_shifted = torch.cat([torch.ones_like(alphas[:, :1]), 1 - alphas + 1e-10], -1)
    T = torch.cumprod(alphas_shifted, -1)
    weights = alphas * T[:, :-1]
    rgb_final = torch.sum(weights.unsqueeze(-1) * rgbs, -2)
    depth_final = torch.sum(weights * z_samp, -1)
    if white_bkgd:
        pix_alpha = weights.sum(dim=1)
        rgb_final = rgb_final + 1 - pix_alpha.unsqueeze(-1)
    return weights, rgb_final, depth_final


def composite(rays, z_samp, sb, state, latent, w, NS, white_bkgd, eval_batch_size=50000):
    """nerf.py:163-249 including the point-chunk loop (:195-216)."""
    B, K = z_samp.shape
    points = rays[:, None, :3] + z_samp.unsqueeze(2) * rays[:, None, 3:6]
    points = points.reshape(sb, -1, 3)
    viewdirs = rays[:, None, 3:6].expand(-1, K, -1).reshape(sb, -1, 3)
    chunk = (eval_batch_size - 1) // sb + 1
    vals = []
    for p, d in zip(torch.split(points, chunk, dim=1), torch.split(viewdirs, chunk, dim=1)):
        vals.append(field_eval(p, d, state, latent, w, NS))
    out = torch.cat(vals, dim=1).reshape(B, K, -1)
    return composite_from_field(rays, z_samp, out, white_bkgd)


def render(rays, noise, state, latent, w_coarse, w_fine, NS, n_coarse, n_fine, n_fine_depth,
           depth_std=0.01, white_bkgd=True, eval_batch_size=50000):
    """NeRFRenderer.forward (nerf.py:251-303).  rays (SB,B,8); noise = the four draws of
    SURVEY A.6 with B := SB*B rows.  Returns dict(coarse=..., fine=...) of
    (weights (SB*B,K), rgb (SB*B,3), depth (SB*B,), z (SB*B,K))."""
    sb = rays.shape[0]
    rays = rays.reshape(-1, 8)
    z_coarse = sample_coarse(rays, noise["u_coarse"], n_coarse)
    wc, rgbc, dc = composite(rays, z_coarse, sb, state, latent, w_coarse, NS, white_bkgd,
                             eval_batch_size)
    res = {"coarse": dict(weights=wc, rgb=rgbc, depth=dc, z=z_coarse)}
    if n_fine > 0:
        samps = [z_coarse]
        if n_fine - n_fine_depth > 0:
            # the coarse weights are detached (nerf.py:286); the coarse depth below is NOT (nerf.py:289-291), so in
            # grad mode the fine loss also reaches the coarse MLP through the depth-centred samples
            samps.append(sample_fine(rays, wc.detach(), noise["u_fine"], noise["u_fine_jit"], n_coarse))
        if n_fine_depth > 0:
            samps.append(sample_fine_depth(rays, dc, noise["n_depth"], depth_std))
        z_comb, _ = torch.sort(torch.cat(samps, dim=-1), dim=-1)
        wf = w_fine if w_fine is not None else w_coarse
        wts, rgbf, df = composite(rays, z_comb, sb, state, latent, wf, NS, white_bkgd,
                                  eval_batch_size)
        res["fine"] = dict(weights=wts, rgb=rgbf, depth=df, z=z_comb)
    return res


# ----------------------------------------------------------------------------------------
# caller-side rows (SURVEY 8f-3): ray generation and frame assembly
# ----------------------------------------------------------------------------------------


def gen_rays(poses, width, height, fx, fy, cx, cy, z_near, z_far):
    """util.gen_rays + unproj_map with ndc=False (src/util/util.py:238-276, :113-143).
    poses (NV,4,4) camera-to-world -> (NV,H,W,8) [origin, unit direction, near, far]."""
    ys = (torch.arange(height, dtype=torch.float32) - float(cy)) / float(fy)     # util.py:134-139
    xs = (torch.arange(width, dtype=torch.float32) - float(cx)) / float(fx)
    X = xs[None, :].expand(height, width)
    Y = ys[:, None].expand(height, width)
    cam = torch.stack((X, -Y, -torch.ones_like(X)), dim=-1)                       # :141
    cam = cam / torch.norm(cam, dim=-1).unsqueeze(-1)                             # :142
    nv = poses.shape[0]
    dirs = torch.matmul(poses[:, None, None, :3, :3], cam[None].expand(nv, -1, -1, -1).unsqueeze(-1))[..., 0]
    origins = poses[:, None, None, :3, 3].expand(-1, height, width, -1)          # util.py:251-254
    near = torch.full((nv, height, width, 1), float(z_near))
    far = torch.full((nv, height, width, 1), float(z_far))
    return torch.cat((origins, dirs, near, far), dim=-1)                          # :274-276


def train_loss(rays, rgb_gt, noise, state, latent, w_coarse, w_fine, NS, n_coarse, n_fine, n_fine_depth,
               depth_std=0.01, white_bkgd=True, eval_batch_size=50000, lambda_coarse=1.0, lambda_fine=1.0):
    """The differentiable loss of a training step, train/train.py:199-212 with the shipped conf
    (conf/default.conf:60-78: MSE rgb losses, lambda_coarse = lambda_fine = 1):
    `render_par(all_rays, want_weights=True)` then MSE(coarse.rgb, gt) * lc + MSE(fine.rgb, gt) * lf.
    Every function above is plain differentiable torch, so `train_loss(...).backward()` is the oracle for the
    backward pass (SURVEY 8f-1): gradients w.r.t. the MLP weight dicts and `latent`."""
    res = render(rays, noise, state, latent, w_coarse, w_fine, NS, n_coarse, n_fine, n_fine_depth,
                 depth_std=depth_std, white_bkgd=white_bkgd, eval_batch_size=eval_batch_size)
    gt = rgb_gt.reshape(-1, 3)
    loss = F.mse_loss(res["coarse"]["rgb"], gt)
    if "fine" in res:
        loss = loss * lambda_coarse + F.mse_loss(res["fine"]["rgb"], gt) * lambda_fine
    return loss


def frames_u8(rgb):
    """Frame assembly of eval/gen_video.py:213-222 and :236: `(frames.cpu().numpy() * 255).astype(np.uint8)`,
    i.e. an fp32 multiply and a truncating cast.  rgb: float32 tensor -> uint8 numpy array of the same shape.
    Defined for values in [0, 256/255) only (the cast is implementation-defined outside)."""
    import numpy as np
    return (rgb.detach().cpu().numpy().astype(np.float32) * 255).astype(np.uint8)


# ------------------------------------------------------------------------------------------
# encode() state fixture (tests/golden/encode_state.npz): a seeded model state and scene that the reference and this
# package can both load, so the reference's encode() outputs can be stored without storing the trunk's weights
# ------------------------------------------------------------------------------------------
ENCODE_CASES = {"pool": (True, (2, 2, 48, 64)), "nopool": (False, (1, 3, 40, 40))}
ENCODE_SAMPLES = 4096


def seeded_state(template, seed):
    """A state_dict with the keys and shapes of `template`, filled from a generator in key order: weights ~ N(0, 1/fan_in),
    BatchNorm affine near (1, 0), running stats away from their (0, 1) initial values so eval-mode BN does real work."""
    g = torch.Generator().manual_seed(seed)
    out = {}
    for k in sorted(template):
        t = template[k]
        if not t.is_floating_point():
            out[k] = t.clone()
        elif k.endswith("running_var"):
            out[k] = torch.rand(t.shape, generator=g) + 0.5
        elif k.endswith("running_mean") or k.endswith("bias"):
            out[k] = torch.randn(t.shape, generator=g) * 0.1
        elif t.dim() == 1:                                   # BatchNorm weight
            out[k] = 1.0 + torch.randn(t.shape, generator=g) * 0.1
        else:
            fan_in = t[0].numel()
            out[k] = torch.randn(t.shape, generator=g) / math.sqrt(fan_in)
    return out


def encode_scene(seed, SB, NS, H, W):
    """images (SB,NS,3,H,W) in [-1,1], c2w poses, focal (SB,2), c (SB,2) and index() query points uv (SB*NS,33,2)."""
    g = torch.Generator().manual_seed(seed)
    images = torch.rand(SB, NS, 3, H, W, generator=g) * 2 - 1
    poses = torch.eye(4).repeat(SB, NS, 1, 1)
    poses[..., :3, :3] = torch.linalg.qr(torch.randn(SB, NS, 3, 3, generator=g))[0]
    poses[..., :3, 3] = torch.randn(SB, NS, 3, generator=g)
    focal = torch.rand(SB, 2, generator=g) * 50 + 40
    c = torch.rand(SB, 2, generator=g) * 4 + torch.tensor([W / 2.0, H / 2.0])
    uv = torch.rand(SB * NS, 33, 2, generator=g) * torch.tensor([W * 1.2, H * 1.2]) - 3.0
    return images, poses, focal, c, uv


def encode_sample_index(numel, seed):
    """Fixed positions at which the fixture stores the (large) latent / index() outputs."""
    g = torch.Generator().manual_seed(seed)
    return torch.randperm(numel, generator=g)[:ENCODE_SAMPLES]
