"""pnr_mgpu_render_backward_cam (csrc/pnr_mgpu.cu: the sharded backward of `bind_parallel(net, gpus)` with gradients of
the rays and the source cameras) on the host emulator, over the device lists of tests/test_emu_mgpu_backward.py.  The
camera gradients sit in each shard's gradient arena and must equal, bit for bit, n separate pnr_render_backward_cam
calls over the same ray slices summed in shard order; the ray gradients must equal the per-shard results put back in
ray order, bit for bit."""
import ctypes as C

import pytest
import torch

import aux_grad_util as au
import emu_util as eu
import golden_util as gu
from test_emu_mgpu_backward import DEVICE_LISTS, _Case, _Sharded, _upstream

pn = eu.pn
rel = au.rel


def _arena(st, want_latent=True):
    """st.arena() followed by the camera gradients (poses, focal, c) -> (flat, coarse struct, fine struct, latent view,
    (d_poses, d_focal, d_c) views)."""
    case, d_h = st.case, st.case["cfg"]["d_hidden"]
    state = gu.oracle_state(case)
    V, Cc, Hl, Wl = case["latent"].shape
    shapes = [v.shape for v in case["wc"].values()] + [v.shape for v in case["wf"].values()]
    if want_latent:
        shapes.append((V, Hl, Wl, Cc))
    shapes += [state["poses"].shape, state["focal"].shape, state["c"].shape]
    flat = torch.zeros(sum(torch.Size(s).numel() for s in shapes))
    views, off = [], 0
    for s in shapes:
        n = torch.Size(s).numel()
        views.append(flat[off:off + n].view(s))
        off += n
    nc = len(case["wc"])
    g_c = dict(zip(case["wc"].keys(), views[:nc]))
    g_f = dict(zip(case["wf"].keys(), views[nc:2 * nc]))
    lat = views[2 * nc] if want_latent else None
    cam = tuple(views[-3:])
    return flat, eu.mlp_struct(g_c, d_h), eu.mlp_struct(g_f, d_h), lat, cam


def _cam_struct(cam, keep):
    keep.append(cam)
    return pn.PnrCameraGrad(*(eu.ptr(t) for t in cam))


def _single(st, a, b, up):
    """pnr_render_backward_cam over rays [a, b) of every object into a fresh arena -> (flat, d_rays [SB][b-a][8])."""
    keep = []
    flat, gsc, gsf, d_lat, cam = _arena(st)
    fwd = pn.PnrRenderOut()
    fwd_t = {k: st.rows(st.t[k], a, b) for k in ("z_coarse", "z_fine", "depth_coarse")}
    fwd.z_coarse, fwd.z_fine, fwd.depth_coarse = (eu.ptr(fwd_t["z_coarse"]), eu.ptr(fwd_t["z_fine"]),
                                                  eu.ptr(fwd_t["depth_coarse"]))
    ug = pn.PnrRenderGrad()
    ups = {k: st.rows(v, a, b) for k, v in up.items()}
    for k, v in ups.items():
        setattr(ug, k, eu.ptr(v))
    rays = st.rays[:, a:b].contiguous()
    d_rays = torch.full((st.SB, b - a, 8), float("nan"))
    L = eu.lib()
    Bi = b - a
    nbytes = L.pnr_render_backward_workspace_bytes(st.scene, st.mc, st.mf, st.rc, Bi)
    ws = torch.empty(nbytes, dtype=torch.uint8)
    nz = {k: st.rows(v, a, b) for k, v in st.nz.items()}
    eu.ok(L.pnr_render_backward_cam(st.scene, st.mc, st.mf, st.rc, eu.ptr(rays), st.noise(nz), fwd, ug, gsc, gsf,
                                    eu.ptr(d_lat), eu.ptr(d_rays), C.byref(_cam_struct(cam, keep)), Bi,
                                    ws.data_ptr(), nbytes, None))
    return flat, d_rays


def _sharded(sh, up, rays=True, cam=True, break_cams=None):
    """The driver's backward with ray / camera gradients -> (rc, flat0, d_rays0, cam0 views)."""
    st, n, L = sh.st, sh.n, eu.lib()
    keep = []
    sgs = (pn.PnrShardGrad * n)()
    scs = (pn.PnrShardCam * n)()
    flat0, gsc0, gsf0, d_lat0, cam0 = _arena(st)
    for i, (a, b) in enumerate(sh.bounds):
        Bi = b - a
        if Bi <= 0:
            continue
        t, _ = sh.stage[i]
        sg = sgs[i]
        rays_i = sh.shard_rays(i).contiguous()
        sg.rays, sg.z_coarse, sg.z_fine, sg.depth_coarse = (eu.ptr(rays_i), eu.ptr(t["z_coarse"]),
                                                            eu.ptr(t["z_fine"]), eu.ptr(t["depth_coarse"]))
        up_stage = torch.full((st.SB * Bi * (8 + 2 * st.Kc + st.Kf),), float("nan"))
        sg.up_stage = eu.ptr(up_stage)
        wsb = L.pnr_render_backward_workspace_bytes(st.scene, st.mc, st.mf, st.rc, Bi)
        ws = torch.empty(wsb, dtype=torch.uint8)
        sg.workspace, sg.workspace_bytes = ws.data_ptr(), wsb
        dr = torch.full((st.SB, Bi, 8), float("nan"))
        scs[i].d_rays = eu.ptr(dr)
        keep += [rays_i, up_stage, ws, dr]
        if i == 0:
            sg.arena, sg.arena_count = eu.ptr(flat0), flat0.numel()
            continue
        flat, gsc, gsf, d_lat, cams = _arena(st)
        flat.fill_(float("nan"))                        # the driver zeroes the shards' arenas
        sg.grad_coarse, sg.grad_fine, sg.d_latent_nhwc = C.pointer(gsc), C.pointer(gsf), eu.ptr(d_lat)
        sg.arena, sg.arena_count = eu.ptr(flat), flat.numel()
        scs[i].cam = _cam_struct(cams, keep)
        if not L.pnr_mgpu_peer_load(sh.h, i):
            stage0 = torch.full_like(flat, float("nan"))
            sg.arena_stage0 = eu.ptr(stage0)
            keep.append(stage0)
        keep += [flat, gsc, gsf]
    if break_cams is not None:
        break_cams(scs, keep)
    ug = pn.PnrRenderGrad()
    for k, v in up.items():
        setattr(ug, k, eu.ptr(v))
    d_rays0 = torch.full((st.SB, st.B, 8), float("nan")) if rays else None
    c0 = C.byref(_cam_struct(cam0, keep)) if cam else None
    rc = L.pnr_mgpu_render_backward_cam(sh.h, sh.shards, sgs, scs, st.rc, ug, gsc0, gsf0, eu.ptr(d_lat0),
                                        eu.ptr(d_rays0), c0, st.B, None)
    return rc, flat0, d_rays0, cam0


@pytest.mark.parametrize("devices", list(DEVICE_LISTS))
@pytest.mark.parametrize("name", gu.GRAD_CASE_NAMES)
def test_sharded_camera_and_ray_gradients_equal_separate_calls(name, devices):
    st = _Case(name)
    up = _upstream(st, name, "all")
    sh = _Sharded(st, DEVICE_LISTS[devices])
    rc, flat, d_rays, cam = _sharded(sh, up)
    eu.ok(rc)
    sh.close()
    total, parts = None, []
    for a, b in sh.bounds:
        if b - a <= 0:
            continue
        f, dr = _single(st, a, b, up)
        total = f if total is None else total + f
        parts.append(dr)
    assert all(t.abs().max() > 0 for t in cam)
    assert torch.equal(flat, total)                                  # weights, latent and cameras, shard order
    assert torch.equal(d_rays, torch.cat(parts, dim=1))
    whole, whole_rays = _single(st, 0, st.B, up)                     # one call: up to the summation order
    assert torch.equal(d_rays, whole_rays)
    assert rel(flat, whole) <= 1e-5


def test_null_requests_are_the_plain_driver_call():
    """With d_rays0 and cam0 NULL, pnr_mgpu_render_backward_cam is pnr_mgpu_render_backward, bit for bit."""
    st = _Case("sb2_d")
    up = _upstream(st, "sb2_d", "all")
    sh = _Sharded(st, [0, 1, 2])
    rc, (flat_a, _, _, _) = sh.backward(up)
    eu.ok(rc)
    rc, flat_b, _, _ = _sharded(sh, up, rays=False, cam=False)
    eu.ok(rc)
    sh.close()
    n = flat_a.numel()
    assert torch.equal(flat_a, flat_b[:n]) and torch.all(flat_b[n:] == 0)


def test_argument_errors():
    st = _Case("sb2_d")
    up = _upstream(st, "sb2_d", "all")
    sh = _Sharded(st, [0, 1])
    L = eu.lib()

    def no_ray_stage(scs, keep):
        scs[1].d_rays = None
    rc, *_ = _sharded(sh, up, break_cams=no_ray_stage)
    assert rc != 0 and b"staging" in L.pnr_last_error()

    def outside_arena(scs, keep):
        t = torch.zeros(64)
        keep.append(t)
        scs[1].cam.d_poses = eu.ptr(t)
    rc, *_ = _sharded(sh, up, break_cams=outside_arena)
    assert rc != 0 and b"arena" in L.pnr_last_error()
    sh.close()
