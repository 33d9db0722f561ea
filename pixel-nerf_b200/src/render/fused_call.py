"""Setup of the fused render call (include/pnr.h: `pnr_render`, `pnr_mgpu_render`) for every caller: inference on one
GPU (`NeRFRenderer._forward_fused`) or sharded (`_ShardedRender`, render/nerf.py), and the training nodes of
render/fused_train.py.  This module alone fills `PnrRenderCfg`, `PnrNoise`, `PnrRenderOut` and `PnrShard`, so the rules
of the C ABI (sample counts, the draws and their order, which outputs exist, what a shard stages) are written once."""
import ctypes as C

import torch

import pnr_native as pn

from .dotmap_compat import DotMap
from .sharding import shard_bounds


def sample_counts(renderer):
    """(Kc, Kf, Kfd, fine) of a call with the renderer's current counts; Kf = Kfd = 0 when the fine pass is off."""
    Kc, Kf, Kfd = int(renderer.n_coarse), int(renderer.n_fine), int(renderer.n_fine_depth)
    if bool(renderer.using_fine) and Kf > 0:
        return Kc, Kf, Kfd, True
    return Kc, 0, 0, False


def render_cfg(renderer, engine):
    Kc, Kf, Kfd, _ = sample_counts(renderer)
    return pn.PnrRenderCfg(Kc, Kf, Kfd, float(renderer.depth_std), 1 if renderer.white_bkgd else 0, pn.ENGINES[engine])


def draw_noise(R, counts, device, noise_in=None, rows=None):
    """The random draws of R rays as fp32 contiguous tensors on `device` -> dict(u_coarse, [u_fine, u_fine_jit],
    [n_depth]), holding only the draws `counts` uses.  Without `noise_in` they are drawn from `device`'s generator in the
    reference's order (nerf.py:111,135,141,158).  With it, its tensors are replayed (tests inject a fixture's draws);
    rows=(SB, B, a, b) then takes from draws of SB * B rays only the rows of rays [a, b) of each object (one shard)."""
    Kc, Kf, Kfd, _ = counts
    f32 = dict(dtype=torch.float32, device=device)
    if noise_in is None:
        draws = {"u_coarse": torch.rand(R, Kc, **f32)}
        if Kf - Kfd > 0:
            draws["u_fine"], draws["u_fine_jit"] = torch.rand(R, Kf - Kfd, **f32), torch.rand(R, Kf - Kfd, **f32)
        if Kfd > 0:
            draws["n_depth"] = torch.randn(R, Kfd, **f32)
        return draws
    names = ["u_coarse"] + (["u_fine", "u_fine_jit"] if Kf - Kfd > 0 else []) + (["n_depth"] if Kfd > 0 else [])
    draws = {}
    for k in names:
        v = noise_in[k]
        if rows is not None:
            SB, B, a, b = rows
            v = v.reshape(SB, B, -1)[:, a:b].flatten(0, 1)
        draws[k] = v.to(**f32).contiguous()
    return draws


def bind_noise(lin_steps, draws):
    """PnrNoise pointing at `lin_steps` and the tensors of `draws`; draws it does not hold stay NULL."""
    noise = pn.PnrNoise()
    noise.lin_steps = pn.dptr(lin_steps)
    for k, t in draws.items():
        setattr(noise, k, pn.dptr(t))
    return noise


def bind_outputs(res):
    """PnrRenderOut pointing at the tensors of `res` (DotMap pass -> quantity -> tensor); fields without one stay NULL."""
    out = pn.PnrRenderOut()
    for field, _ in out._fields_:
        q, p = field.split("_")                  # "weights_fine" -> res.fine.weights
        if p in res and q in res[p]:
            setattr(out, field, pn.dptr(res[p][q]))
    return out


def render_outputs(SB, B, counts, device, want_weights, want_z):
    """Output tensors of a call on SB objects x B rays -> (PnrRenderOut, DotMap(coarse=DotMap(rgb, depth[, weights]
    [, z]), fine=...)), tensors (SB, B, ...) on `device`, fine only with a fine pass; the struct points at them."""
    Kc, Kf, _, fine = counts
    f32 = dict(dtype=torch.float32, device=device)
    res = DotMap()
    for p, K in [("coarse", Kc)] + ([("fine", Kc + Kf)] if fine else []):
        d = DotMap(rgb=torch.empty(SB, B, 3, **f32), depth=torch.empty(SB, B, **f32))
        if want_weights:
            d.weights = torch.empty(SB, B, K, **f32)
        if want_z:
            d.z = torch.empty(SB, B, K, **f32)
        res[p] = d
    return bind_outputs(res), res


def setup_shards(sharded, rays0, counts, cfg, want_weights, want_z, noise_in=None):
    """One PnrShard per GPU of `sharded` (render/nerf.py::_ShardedRender) for rays0 (SB, B, 8) on gpus[0].  Shard i
    gets torch.chunk piece i of the rays along dim 1 and renders it from gpus[i]'s scene: the net itself on gpus[0],
    a `_SceneReplica`, refreshed here, elsewhere.  It draws from gpus[i]'s generator, or takes its rows of
    `noise_in`, and its outputs (with the sample depths when `want_z`, which the backward reads) are staged on gpus[i].
    -> (shards, {i: (stage DotMap, the shard's rays on gpus[i]) for every non-empty shard}, buffers the call reads,
    which must stay referenced until the shards' streams are done with them)."""
    net, renderer = sharded.module.net, sharded.module.renderer
    Kc, _, _, fine = counts
    SB, B, _ = rays0.shape
    L = pn.lib()
    shards = (pn.PnrShard * len(sharded.gpus))()
    stages, keep = {}, [rays0]
    for i, (g, (a, b)) in enumerate(zip(sharded.gpus, shard_bounds(B, len(sharded.gpus)))):
        Bi = b - a
        if Bi <= 0:
            continue
        dev = torch.device("cuda", g)
        model = net
        if i > 0:
            model = sharded._replicas[g]
            sharded._refresh(model, fine)
        with torch.cuda.device(dev):
            scene, mc, mf, keep2 = model._scene_struct(want_fine=fine)
            lin = renderer._lin_steps(Kc, dev)
            draws = draw_noise(SB * Bi, counts, dev, noise_in, rows=(SB, B, a, b))
            noise = bind_noise(lin, draws)
            stage, stage_res = render_outputs(SB, Bi, counts, dev, want_weights, want_z)
            ws = pn.workspace(dev, L.pnr_render_workspace_bytes(scene, mc, mf, cfg, Bi))
            sh = shards[i]
            sh.scene, sh.mlp_coarse = C.pointer(scene), C.pointer(mc)
            sh.mlp_fine = C.pointer(mf) if mf is not None else None
            sh.noise = C.pointer(noise)
            sh.workspace, sh.workspace_bytes = ws.data_ptr(), ws.numel()
            rays_i = rays0
            if i > 0 or SB > 1:
                rays_i = torch.empty(SB, Bi, 8, dtype=torch.float32, device=dev)
                sh.rays_stage = pn.dptr(rays_i)
            sh.stage = stage
            sh.stream = pn.stream_ptr(dev)
            stages[i] = (stage_res, rays_i)
            keep += [lin, draws, keep2, scene, mc, mf, noise, ws, stage_res, rays_i]
    return shards, stages, keep
