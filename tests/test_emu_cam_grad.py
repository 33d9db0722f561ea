"""Gradients w.r.t. the rays and the source cameras through the C ABI, CUDA sources executed on the CPU by the host
emulator of tests/cuda_emu: `pnr_render_backward_cam`, `pnr_field_backward_cam` and `pnr_gen_rays_backward` against
torch autograd through the oracle's forward (oracle/pnr_oracle.py, which restates the reference's differentiable
graph op by op), and the NULL-request calls against the entry points they extend, bit for bit."""
import ctypes as C
import os

import pytest
import torch

import aux_grad_util as au
import emu_render_util as eru
import emu_util as eu
import golden_util as gu

rel = au.rel
pn = eu.pn
OUTS = [(p, q) for p in ("coarse", "fine") for q in ("rgb", "depth", "weights")]


_case = eru.case_with_state
_Render = eru.Render


def _random_up(case, seed, outputs=None):
    cfg = case["cfg"]
    R, Kc, K = cfg["SB"] * cfg["B"], cfg["n_coarse"], cfg["n_coarse"] + cfg["n_fine"]
    g = torch.Generator().manual_seed(seed)
    shapes = dict(rgb=(3,), depth=(), weights_coarse=(Kc,), weights_fine=(K,))
    up = {}
    for p, q in OUTS:
        if p == "fine" and cfg["n_fine"] == 0:
            continue
        if outputs is not None and (p, q) not in outputs:
            continue
        shape = shapes.get(f"{q}_{p}", shapes.get(q))
        up[f"d_{q}_{p}"] = torch.randn(R, *shape, generator=g) * 1e-2
    return up


def _autograd(case, up):
    """Autograd through the oracle's forward: gradients of rays, world->camera poses, focal and c."""
    cfg, st = case["cfg"], case["state"]
    rays = case["rays"].clone().requires_grad_(True)
    state = dict(st)
    for k in ("poses", "focal", "c"):
        state[k] = st[k].clone().requires_grad_(True)
    res = gu.oracle.render(rays, case["noise"], state, case["latent"], case["wc"], case["wf"], cfg["NS"],
                           cfg["n_coarse"], cfg["n_fine"], cfg["n_fine_depth"], depth_std=cfg["depth_std"],
                           white_bkgd=bool(cfg["white_bkgd"]), eval_batch_size=cfg["eval_batch_size"])
    outs, grads = [], []
    for p, q in OUTS:
        if f"d_{q}_{p}" in up:
            outs.append(res[p][q])
            grads.append(up[f"d_{q}_{p}"])
    torch.autograd.backward(outs, grad_tensors=grads)
    z_fine = res["fine"]["z"].detach() if "fine" in res else None
    return dict(rays=rays.grad.reshape(-1, 8), poses=state["poses"].grad, focal=state["focal"].grad,
                c=state["c"].grad), z_fine


def _check(case, up, tol=2e-4):
    step = _Render(case)
    ref, z_fine = _autograd(case, up)
    if z_fine is not None:     # the comparison needs identical samples
        assert (step.t["z_fine"] - z_fine).abs().max() < 1e-5
    got = step.backward(up, rays=True, cam=True)
    for k in ("rays", "poses", "focal", "c"):
        assert ref[k].abs().max() > 0, k
        assert rel(got[k], ref[k]) < tol, (k, rel(got[k], ref[k]))
    return step, got


@pytest.mark.parametrize("name", ["tiny", "sb2_d", "ns1_coarse_only"])
def test_render_backward_cam_matches_autograd(name):
    case = _case(name)
    _check(case, _random_up(case, 3))


@pytest.mark.parametrize("name", gu.GRAD_CASE_NAMES)
def test_render_backward_cam_on_the_reference_upstream_gradients(name):
    """The upstream gradients the reference's all-outputs loss produced (tests/golden/grad_aux_*.npz)."""
    case = _case(name)
    _check(case, au.flat_up(au.load(name), case["cfg"]["SB"] * case["cfg"]["B"]))


@pytest.mark.parametrize("n_fine,n_fine_depth,depth_std", [(0, 0, 0.01), (6, 0, 0.01), (6, 3, 0.6), (4, 4, 0.6)])
def test_render_backward_cam_edge_cases(n_fine, n_fine_depth, depth_std):
    """Coarse only, no depth-centred samples, and depth-centred samples of which many clamp to near or far; per-object
    focal and c (SB = 2)."""
    case = _case("sb2_d", n_fine, n_fine_depth, depth_std=depth_std, per_object_c=True, seed=n_fine + n_fine_depth)
    cfg = case["cfg"]
    assert case["state"]["focal"].shape[0] == case["state"]["c"].shape[0] == cfg["SB"] == 2
    if n_fine_depth > 0:
        step = _Render(case)
        rays = case["rays"].reshape(-1, 8)
        zz = step.t["depth_coarse"][:, None] + case["noise"]["n_depth"] * depth_std
        assert (zz > rays[:, 7:8]).any() and (zz < rays[:, 6:7]).any()
    _check(case, _random_up(case, 5 + n_fine))


@pytest.mark.parametrize("outputs", [[("fine", "depth")], [("coarse", "rgb")], [("fine", "weights")]])
def test_render_backward_cam_with_one_output_gradient(outputs):
    """Only one pass carries an upstream gradient: d_rays is still fully written."""
    case = _case("sb2_d")
    _check(case, _random_up(case, 9, outputs))


@pytest.mark.parametrize("name", ["tiny", "sb2_d", "ns1_coarse_only"])
def test_null_requests_are_the_ex_call_bit_for_bit(name):
    case = _case(name)
    step = _Render(case)
    up = _random_up(case, 1)
    a = step.backward(up, entry="ex")
    b = step.backward(up, entry="cam")
    c = step.backward(up, rays=True, cam=True)
    assert a["launches"] == b["launches"] and c["launches"] > a["launches"]
    assert torch.equal(a["lat"], b["lat"]) and torch.equal(a["lat"], c["lat"])
    for key in ("gc", "gf"):
        for k in (a[key] or {}):
            assert torch.equal(a[key][k], b[key][k]), (key, k)
            assert torch.equal(a[key][k], c[key][k]), (key, k)


def test_render_backward_cam_is_deterministic():
    case = _case("sb2_d")
    step = _Render(case)
    up = _random_up(case, 2)
    a, b = step.backward(up, rays=True, cam=True), step.backward(up, rays=True, cam=True)
    for k in ("rays", "poses", "focal", "c"):
        assert torch.equal(a[k], b[k]), k


def _field_call(case, xyz, dirs, d_out, with_new=True, chunk_rows=None):
    cfg, st = case["cfg"], case["state"]
    keep = []
    scene = eu.scene_struct(case, st, keep)
    wc = case["wc"]
    m = eu.mlp_struct(wc, cfg["d_hidden"])
    g = {k: torch.zeros_like(v) for k, v in wc.items()}
    gs = eu.mlp_struct(g, cfg["d_hidden"])
    SB, P, _ = xyz.shape
    L = eu.lib()
    nbytes = L.pnr_field_backward_workspace_bytes(scene, m, P)
    ws = torch.empty(nbytes, dtype=torch.uint8)
    d_xyz = torch.empty(SB, P, 3)
    V, Cc, Hl, Wl = case["latent"].shape
    d_lat = torch.zeros(V, Hl, Wl, Cc)
    out = dict(g=g, lat=d_lat, xyz=d_xyz)
    if with_new:
        out.update(dirs=torch.full((SB, P, 3), float("nan")), poses=torch.zeros_like(st["poses"]),
                   focal=torch.zeros_like(st["focal"]), c=torch.zeros_like(st["c"]))
        cg = pn.PnrCameraGrad(eu.ptr(out["poses"]), eu.ptr(out["focal"]), eu.ptr(out["c"]))
        eu.ok(L.pnr_field_backward_cam(scene, m, eu.ptr(xyz), eu.ptr(dirs), eu.ptr(d_out), gs, eu.ptr(d_lat),
                                       eu.ptr(d_xyz), eu.ptr(out["dirs"]), C.byref(cg), P, ws.data_ptr(), nbytes,
                                       None))
    else:
        eu.ok(L.pnr_field_backward(scene, m, eu.ptr(xyz), eu.ptr(dirs), eu.ptr(d_out), gs, eu.ptr(d_lat),
                                   eu.ptr(d_xyz), P, ws.data_ptr(), nbytes, None))
    return out


def _field_inputs(case, P, seed):
    cfg = case["cfg"]
    g = torch.Generator().manual_seed(seed)
    rays = case["rays"].reshape(cfg["SB"], -1, 8)
    idx = torch.randint(0, rays.shape[1], (P,), generator=g)
    r = rays[:, idx]
    z = 0.8 + torch.rand(cfg["SB"], P, 1, generator=g)
    xyz = (r[..., :3] + z * r[..., 3:6]).contiguous()
    dirs = r[..., 3:6].contiguous()
    d_out = (torch.randn(cfg["SB"], P, 4, generator=g) * 1e-2).contiguous()
    return xyz, dirs, d_out


@pytest.mark.parametrize("name,chunk_rows", [("sb2_d", None), ("tiny", None), ("sb2_d", "10")])
def test_field_backward_cam_matches_autograd(name, chunk_rows, monkeypatch):
    """Also split into several point chunks (the per-view reduction runs once per chunk)."""
    case = _case(name, per_object_c=(name == "sb2_d"))
    cfg, st = case["cfg"], case["state"]
    xyz, dirs, d_out = _field_inputs(case, 29, 4)
    if chunk_rows:
        monkeypatch.setenv("PNR_BWD_CHUNK_ROWS", chunk_rows)
    got = _field_call(case, xyz, dirs, d_out)
    x, d = xyz.clone().requires_grad_(True), dirs.clone().requires_grad_(True)
    state = dict(st)
    for k in ("poses", "focal", "c"):
        state[k] = st[k].clone().requires_grad_(True)
    gu.oracle.field_eval(x, d, state, case["latent"], case["wc"], cfg["NS"]).backward(d_out)
    assert rel(got["xyz"], x.grad) < 2e-4
    assert rel(got["dirs"], d.grad) < 2e-4
    for k in ("poses", "focal", "c"):
        assert rel(got[k], state[k].grad) < 2e-4, k
    ref = _field_call(case, xyz, dirs, d_out, with_new=False)
    assert torch.equal(ref["xyz"], got["xyz"]) and torch.equal(ref["lat"], got["lat"])
    for k in ref["g"]:
        assert torch.equal(ref["g"][k], got["g"][k]), k


@pytest.mark.parametrize("first,count", [(0, 2 * 7 * 5), (13, 40), (35, 1), (3, 100)])
def test_gen_rays_backward_matches_autograd(first, count):
    g = torch.Generator().manual_seed(first)
    NV, W, H = 3, 7, 5
    poses = torch.eye(4).repeat(NV, 1, 1)
    poses[:, :3, :3] = torch.linalg.qr(torch.randn(NV, 3, 3, generator=g))[0]
    poses[:, :3, 3] = torch.randn(NV, 3, generator=g)
    fx, fy, cx, cy = 6.5, 7.25, 3.1, 2.4
    p = poses.clone().requires_grad_(True)
    rays = gu.oracle.gen_rays(p, W, H, fx, fy, cx, cy, 0.5, 2.0).reshape(-1, 8)[first:first + count]
    d_rays = torch.randn(count, 8, generator=g)
    rays.backward(d_rays)
    got = torch.full((NV, 4, 4), 0.25)
    eu.ok(eu.lib().pnr_gen_rays_backward(eu.ptr(d_rays), eu.ptr(poses), NV, W, H, fx, fy, cx, cy, first, count,
                                         eu.ptr(got), None))
    assert rel(got - 0.25, p.grad) < 1e-5
    assert torch.all(got[:, 3] == 0.25)


def test_argument_errors():
    L = eu.lib()
    d = torch.zeros(4, 8)
    p = torch.zeros(1, 4, 4)
    assert L.pnr_gen_rays_backward(eu.ptr(d), eu.ptr(p), 1, 2, 2, 1.0, 1.0, 0.0, 0.0, 1, 4, eu.ptr(p), None) != 0
    assert b"outside" in L.pnr_last_error()
    assert L.pnr_gen_rays_backward(None, eu.ptr(p), 1, 2, 2, 1.0, 1.0, 0.0, 0.0, 0, 4, eu.ptr(p), None) != 0
    assert L.pnr_gen_rays_backward(eu.ptr(d), eu.ptr(p), 1, 2, 2, 0.0, 1.0, 0.0, 0.0, 0, 4, eu.ptr(p), None) != 0
    case = _case("tiny")
    step = _Render(case)
    nbytes = L.pnr_render_backward_workspace_bytes(step.scene, step.mc, step.mf, step.rc, case["cfg"]["B"])
    ws = torch.empty(nbytes - 1024, dtype=torch.uint8)
    gs = eu.mlp_struct({k: torch.zeros_like(v) for k, v in case["wc"].items()}, case["cfg"]["d_hidden"])
    d_rays = torch.zeros(step.R, 8)
    rc = L.pnr_render_backward_cam(step.scene, step.mc, step.mf, step.rc, eu.ptr(step.rays), step.noise, step.out,
                                   None, gs, gs, None, eu.ptr(d_rays), None, case["cfg"]["B"], ws.data_ptr(),
                                   ws.numel(), None)
    assert rc != 0 and b"workspace" in L.pnr_last_error()
