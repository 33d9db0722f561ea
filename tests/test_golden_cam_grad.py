"""Ray and camera gradients against the gradients the unmodified reference computed itself
(tests/golden/grad_cam_*.npz, oracle/make_golden_cam.py: rays, camera-to-world source poses, focal and c requiring grad,
a loss on all six outputs): autograd through the oracle, the composed-torch path of this package on the CPU (which
checks that `set_cameras` keeps the graph from encode()'s inputs) and `pnr_render_backward_cam` on the host emulator.
CPU only."""
import copy
import ctypes as C
import os

import numpy as np
import pytest
import torch

import aux_grad_util as au
import emu_util as eu
import golden_util as gu

rel = au.rel
FIXTURES = {"tiny": "tiny", "sb2_d": "sb2_d", "sb2_d_clamp": "sb2_d"}
OUTS = [("coarse", "rgb"), ("coarse", "depth"), ("coarse", "weights"), ("fine", "rgb"), ("fine", "depth"),
        ("fine", "weights")]


def load(fixture):
    z = np.load(os.path.join(gu.GOLD, "grad_cam_" + fixture + ".npz"))
    t = lambda k: torch.from_numpy(z[k])
    return dict(depth_std=float(z["depth_std"]), c=t("c"), up={f"{p}.{q}": t(f"up/{p}.{q}") for p, q in OUTS},
                rays=t("g_rays"), poses=t("g_poses"), focal=t("g_focal"), g_c=t("g_c"), latent=t("g_latent"),
                gc={k[3:]: t(k) for k in z.files if k.startswith("gc/")})


def _leaves(case, fx):
    poses = case["src_poses"].clone().requires_grad_(True)
    focal = case["focal"].clone().float().requires_grad_(True)
    c = fx["c"].clone().requires_grad_(True)
    rays = case["rays"].clone().requires_grad_(True)
    return rays, poses, focal, c


def _check(fx, rays, poses, focal, c, tol):
    for got, ref, k in ((rays.grad, fx["rays"], "rays"), (poses.grad, fx["poses"], "poses"),
                        (focal.grad, fx["focal"], "focal"), (c.grad, fx["g_c"], "c")):
        assert ref.abs().max() > 0, k
        assert rel(got.reshape(ref.shape), ref) < tol, (k, rel(got.reshape(ref.shape), ref))


def test_clamp_fixture_clamps_depth_samples():
    case, fx = gu.load_case("sb2_d"), load("sb2_d_clamp")
    depth = gu.oracle_render(case)["coarse"]["depth"]
    zz = depth[:, None] + case["noise"]["n_depth"] * fx["depth_std"]
    rays = case["rays"].reshape(-1, 8)
    assert (zz > rays[:, 7:8]).any() and (zz < rays[:, 6:7]).any()


@pytest.mark.parametrize("fixture", list(FIXTURES))
def test_oracle_autograd_matches_reference(fixture):
    case, fx = gu.load_case(FIXTURES[fixture]), load(fixture)
    cfg = case["cfg"]
    rays, poses, focal, c = _leaves(case, fx)
    state = gu.oracle.encode_state(poses.reshape(-1, 4, 4), focal, c, cfg["W"], cfg["H"])
    res = gu.oracle.render(rays, case["noise"], state, case["latent"], case["wc"], case["wf"], cfg["NS"],
                           cfg["n_coarse"], cfg["n_fine"], cfg["n_fine_depth"], depth_std=fx["depth_std"],
                           white_bkgd=bool(cfg["white_bkgd"]), eval_batch_size=cfg["eval_batch_size"])
    outs = [res[p][q] for p, q in OUTS]
    torch.autograd.backward(outs, [fx["up"][f"{p}.{q}"].reshape(t.shape) for (p, q), t in zip(OUTS, outs)])
    _check(fx, rays, poses, focal, c, 1e-4)


@pytest.mark.parametrize("fixture", list(FIXTURES))
def test_composed_torch_path_matches_reference(fixture):
    """This package's PixelNeRFNet + NeRFRenderer on the CPU in grad mode (_forward_torch / _forward_autograd), seeded
    as the reference was: the gradients reach encode()'s poses, focal and c through set_cameras."""
    import gpu_util
    case, fx = gu.load_case(FIXTURES[fixture]), load(fixture)
    cfg = case["cfg"]
    net = gpu_util.build_net(case, device="cpu").train().requires_grad_(False)
    rays, poses, focal, c = _leaves(case, fx)
    net.set_scene(case["latent"], poses, focal, c, cfg["W"], cfg["H"])
    renderer = gpu_util.build_renderer(case).train()
    renderer.depth_std = fx["depth_std"]
    torch.manual_seed(case["seed"] + 4)
    out = renderer(net, rays, want_weights=True)
    outs = [out[p][q] for p, q in OUTS]
    torch.autograd.backward(outs, [fx["up"][f"{p}.{q}"].reshape(t.shape) for (p, q), t in zip(OUTS, outs)])
    _check(fx, rays, poses, focal, c, 1e-4)


@pytest.mark.parametrize("fixture", list(FIXTURES))
def test_emulated_render_backward_cam_matches_reference(fixture):
    """pnr_render_backward_cam on the emulator; its world->camera / (fx, -fy) gradients are carried to encode()'s
    inputs by autograd of the oracle's encode_state (models.py:112-141)."""
    import test_emu_cam_grad as ec
    case, fx = gu.load_case(FIXTURES[fixture]), load(fixture)
    cfg = case["cfg"]
    rays, poses, focal, c = _leaves(case, fx)
    state = gu.oracle.encode_state(poses.reshape(-1, 4, 4), focal, c, cfg["W"], cfg["H"])
    case = copy.copy(case)
    case["cfg"] = dict(cfg, depth_std=fx["depth_std"])
    case["state"] = {k: (v.detach().contiguous() if torch.is_tensor(v) else v) for k, v in state.items()}
    up = au.flat_up(dict(up=fx["up"]), cfg["SB"] * cfg["B"])
    step = ec._Render(case)
    got = step.backward(up, rays=True, cam=True)
    torch.autograd.backward([state["poses"], state["focal"], state["c"]], [got["poses"], got["focal"], got["c"]])
    rays.grad = got["rays"].reshape(rays.shape)
    _check(fx, rays, poses, focal, c, 2e-4)
