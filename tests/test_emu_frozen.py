"""Backward of a partly frozen network on the host emulator: `pnr_render_backward_sel`, `pnr_field_backward_sel` and
`pnr_mgpu_render_backward_sel` (NULL gradient structs or members = frozen) against the full `_cam` calls.  Every
gradient the selective call computes must equal, bit for bit, the same tensor of the full call, in fewer launches
whenever something is frozen; with everything wanted the selective call is the full call, launch for launch."""
import copy
import ctypes as C

import pytest
import torch

import emu_util as eu
import golden_util as gu
from test_emu_cam_grad import _Render, _case, _field_inputs, _random_up
from test_emu_mgpu_backward import DEVICE_LISTS, _Case, _Sharded

pn = eu.pn


def _ns3_case():
    """tiny with a third source view (NS = 3): view 0's camera moved a little, looking at view 1's mirrored features."""
    case = copy.copy(gu.load_case("tiny"))
    sp = case["src_poses"]
    extra = sp[:, :1].clone()
    extra[..., :3, 3] += torch.tensor([0.05, -0.03, 0.02])
    case["src_poses"] = torch.cat([sp, extra], dim=1).contiguous()
    case["latent"] = torch.cat([case["latent"], case["latent"][1:2].flip(-1)]).contiguous()
    case["cfg"] = dict(case["cfg"], NS=3, depth_std=0.01)
    case["state"] = gu.oracle_state(case)
    return case


# NS = 1..3, one and two objects, with and without a fine MLP, with and without depth-centred fine samples
CASES = {
    "tiny": lambda: _case("tiny"),                                  # NS 2, fine MLP, depth samples
    "tiny_sb2": lambda: _case("tiny_sb2"),                          # two objects, mlp_fine = None, depth samples
    "sb2_d": lambda: _case("sb2_d"),                                # two objects, fine MLP
    "sb2_d_no_depth": lambda: _case("sb2_d", n_fine=6, n_fine_depth=0),
    "ns1_coarse_only": lambda: _case("ns1_coarse_only"),            # NS 1, no fine pass
    "ns3": _ns3_case,
}

# name -> (is (mlp "c"/"f", parameter name) trainable, (latent, rays, cameras) wanted)
PATTERNS = {
    "network_frozen_rays_poses": (lambda m, k: False, (False, True, True)),
    "encoder_frozen": (lambda m, k: True, (False, False, False)),
    "coarse_frozen": (lambda m, k: m == "f", (True, False, False)),
    "fine_frozen": (lambda m, k: m == "c", (True, False, False)),
    "blocks_3_4_and_lin_out": (lambda m, k: k.startswith(("blocks.3.", "blocks.4.", "lin_out.")), (False, False, False)),
    "lin_in_only": (lambda m, k: k.startswith("lin_in."), (False, False, False)),
    "biases_only": (lambda m, k: k.endswith(".bias"), (False, False, False)),
    "nothing": (lambda m, k: False, (False, False, False)),
}
ALL = (lambda m, k: True, (True, True, True))


def _grads(sd, tag, trainable, d_hidden):
    """Zeroed gradients of the trainable tensors of `sd` -> (dict, PnrMlp with NULL for the rest, or None for none)."""
    if sd is None:
        return None, None
    g = {k: torch.zeros_like(v) for k, v in sd.items() if trainable(tag, k)}
    if not g:
        return g, None
    m = eu.mlp_struct({k: g.get(k, sd[k]) for k in sd}, d_hidden)
    for k in sd:                                                    # NULL every frozen member
        if k not in g:
            _null(m, k)
    return g, m


def _null(m, key):
    parts = key.split(".")
    wb = "w" if parts[-1] == "weight" else "b"
    if parts[0] in ("lin_in", "lin_out"):
        setattr(m, f"{parts[0]}_{wb}", None)
    elif parts[0] == "lin_z":
        getattr(m, f"lin_z_{wb}")[int(parts[1])] = None
    else:                                                           # blocks.i.fc_j
        getattr(m, f"fc{parts[2][-1]}_{wb}")[int(parts[1])] = None


def _render_backward(step, up, pattern, entry):
    """One backward of `step` (test_emu_cam_grad._Render) -> dict(gc, gf, lat, rays, poses, focal, c, launches)."""
    trainable, (lat, rays, cam) = pattern
    case, cfg, st = step.case, step.case["cfg"], step.case["state"]
    g_c, gsc = _grads(case["wc"], "c", trainable, cfg["d_hidden"])
    g_f, gsf = _grads(case["wf"], "f", trainable, cfg["d_hidden"])
    V, Cc, Hl, Wl = case["latent"].shape
    out = dict(gc=g_c, gf=g_f, lat=torch.zeros(V, Hl, Wl, Cc) if lat else None,
               rays=torch.full((step.R, 8), float("nan")) if rays else None)
    cg = None
    if cam:
        out.update(poses=torch.zeros_like(st["poses"]), focal=torch.zeros_like(st["focal"]), c=torch.zeros_like(st["c"]))
        cg = pn.PnrCameraGrad(eu.ptr(out["poses"]), eu.ptr(out["focal"]), eu.ptr(out["c"]))
    ug = pn.PnrRenderGrad()
    up = {k: v.contiguous() for k, v in up.items()}
    for k, v in up.items():
        setattr(ug, k, eu.ptr(v))
    L = eu.lib()
    nbytes = L.pnr_render_backward_workspace_bytes(step.scene, step.mc, step.mf, step.rc, cfg["B"])
    ws = torch.empty(nbytes, dtype=torch.uint8)
    fn = L.pnr_render_backward_sel if entry == "sel" else L.pnr_render_backward_cam
    ref = lambda s: C.byref(s) if s is not None else None
    n0 = L.pnr_launch_count()
    eu.ok(fn(step.scene, step.mc, step.mf, step.rc, eu.ptr(step.rays), step.noise, step.out, ug, ref(gsc), ref(gsf),
             eu.ptr(out["lat"]), eu.ptr(out["rays"]), ref(cg), cfg["B"], ws.data_ptr(), nbytes, None))
    out["launches"] = L.pnr_launch_count() - n0
    return out


def _assert_subset_equal(sel, full):
    """Every tensor `sel` computed equals the same tensor of `full`, bit for bit."""
    for key in ("gc", "gf"):
        for k, v in (sel.get(key) or {}).items():
            assert torch.equal(v, full[key][k]), (key, k)
    for key in ("lat", "rays", "poses", "focal", "c"):
        if sel.get(key) is not None:
            assert torch.equal(sel[key], full[key]), key


@pytest.fixture(scope="module")
def steps():
    return {name: _Render(make()) for name, make in CASES.items()}


@pytest.mark.parametrize("pattern", list(PATTERNS))
@pytest.mark.parametrize("name", list(CASES))
def test_frozen_gradients_equal_the_full_call(steps, name, pattern):
    step = steps[name]
    up = _random_up(step.case, 11)                   # all six outputs carry a gradient: both passes and the depth path
    full = _render_backward(step, up, ALL, "cam")
    sel = _render_backward(step, up, PATTERNS[pattern], "sel")
    _assert_subset_equal(sel, full)
    assert sel["launches"] < full["launches"], (sel["launches"], full["launches"])
    if pattern == "nothing":
        assert sel["launches"] == 0
    trainable = PATTERNS[pattern][0]
    if name == "tiny_sb2":                           # its MLP renders nothing (sigma = 0): all gradients are zero
        return
    for tag, key in (("c", "gc"), ("f", "gf")):
        for k, v in (sel[key] or {}).items():
            if trainable(tag, k) and k.endswith("weight"):
                assert v.abs().max() > 0, (key, k)   # a trainable tensor got a real gradient


@pytest.mark.parametrize("name", list(CASES))
def test_everything_wanted_is_the_full_call(steps, name):
    step = steps[name]
    up = _random_up(step.case, 12)
    full = _render_backward(step, up, ALL, "cam")
    sel = _render_backward(step, up, ALL, "sel")
    assert sel["launches"] == full["launches"]
    _assert_subset_equal(sel, full)


def test_fine_pass_runs_for_the_coarse_depth_when_only_the_coarse_mlp_trains(steps):
    """Only the fine outputs carry a gradient, but their depth-centred samples reach the coarse depth: a trainable
    coarse MLP still needs the fine pass's positions gradient."""
    step = steps["tiny"]
    up = _random_up(step.case, 13, outputs=[("fine", "rgb")])
    full = _render_backward(step, up, ALL, "cam")
    sel = _render_backward(step, up, PATTERNS["fine_frozen"], "sel")
    _assert_subset_equal(sel, full)
    assert sel["gc"]["lin_out.weight"].abs().max() > 0


def _field_backward(case, xyz, dirs, d_out, pattern, entry, want_dirs=False):
    trainable, (lat, want_xyz, cam) = pattern
    cfg, st = case["cfg"], case["state"]
    keep = []
    scene = eu.scene_struct(case, st, keep)
    m = eu.mlp_struct(case["wc"], cfg["d_hidden"])
    g, gs = _grads(case["wc"], "c", trainable, cfg["d_hidden"])
    SB, P, _ = xyz.shape
    V, Cc, Hl, Wl = case["latent"].shape
    out = dict(gc=g, lat=torch.zeros(V, Hl, Wl, Cc) if lat else None, xyz=torch.zeros(SB, P, 3) if want_xyz else None,
               dirs=torch.zeros(SB, P, 3) if want_dirs else None)
    cg = None
    if cam:
        out.update(poses=torch.zeros_like(st["poses"]), focal=torch.zeros_like(st["focal"]), c=torch.zeros_like(st["c"]))
        cg = pn.PnrCameraGrad(eu.ptr(out["poses"]), eu.ptr(out["focal"]), eu.ptr(out["c"]))
    L = eu.lib()
    nbytes = L.pnr_field_backward_workspace_bytes(scene, m, P)
    ws = torch.empty(nbytes, dtype=torch.uint8)
    fn = L.pnr_field_backward_sel if entry == "sel" else L.pnr_field_backward_cam
    n0 = L.pnr_launch_count()
    eu.ok(fn(scene, m, eu.ptr(xyz), eu.ptr(dirs), eu.ptr(d_out), C.byref(gs) if gs is not None else None,
             eu.ptr(out["lat"]), eu.ptr(out["xyz"]), eu.ptr(out["dirs"]), C.byref(cg) if cg is not None else None, P,
             ws.data_ptr(), nbytes, None))
    out["launches"] = L.pnr_launch_count() - n0
    return out


@pytest.mark.parametrize("pattern", list(PATTERNS) + ["viewdirs_only"])
def test_field_backward_sel_over_several_chunks(pattern, monkeypatch):
    """pnr_field_backward_sel with the points split into several chunks (rays slot = d_xyz here); viewdirs_only wants
    nothing but d_viewdirs, which needs the geometry backward without dlat."""
    monkeypatch.setenv("PNR_BWD_CHUNK_ROWS", "10")
    case = _case("sb2_d", per_object_c=True)
    xyz, dirs, d_out = _field_inputs(case, 29, 4)
    full = _field_backward(case, xyz, dirs, d_out, ALL, "cam", want_dirs=True)
    pat = PATTERNS.get(pattern, (lambda m, k: False, (False, False, False)))
    sel = _field_backward(case, xyz, dirs, d_out, pat, "sel", want_dirs=pattern == "viewdirs_only")
    _assert_subset_equal(sel, full)
    for key in ("xyz", "dirs"):
        if sel[key] is not None:
            assert torch.equal(sel[key], full[key]), key
    assert sel["launches"] < full["launches"]
    if pattern == "nothing":
        assert sel["launches"] == 0


def test_sel_argument_errors():
    case = _case("tiny")
    xyz, dirs, d_out = _field_inputs(case, 5, 1)
    keep = []
    scene = eu.scene_struct(case, case["state"], keep)
    m = eu.mlp_struct(case["wc"], case["cfg"]["d_hidden"])
    g, gs = _grads(case["wc"], "c", lambda t, k: True, case["cfg"]["d_hidden"])
    gs.n_blocks = 4
    L = eu.lib()
    nbytes = L.pnr_field_backward_workspace_bytes(scene, m, 5)
    ws = torch.empty(nbytes, dtype=torch.uint8)
    rc = L.pnr_field_backward_sel(scene, m, eu.ptr(xyz), eu.ptr(dirs), eu.ptr(d_out), C.byref(gs), None, None, None,
                                  None, 5, ws.data_ptr(), nbytes, None)
    assert rc != 0 and b"shape" in L.pnr_last_error()
    # the full entry points still require every gradient
    g2, gs2 = _grads(case["wc"], "c", lambda t, k: k != "lin_in.bias", case["cfg"]["d_hidden"])
    rc = L.pnr_field_backward_cam(scene, m, eu.ptr(xyz), eu.ptr(dirs), eu.ptr(d_out), C.byref(gs2), None, None, None,
                                  None, 5, ws.data_ptr(), nbytes, None)
    assert rc != 0 and b"NULL" in L.pnr_last_error()


# ---------------------------------------------------------------------------------------------------------------------
# several devices: pnr_mgpu_render_backward_sel against per-shard pnr_render_backward_sel calls summed in shard order
# ---------------------------------------------------------------------------------------------------------------------
def _sel_arena(st, pattern):
    """Device-0-layout arena holding only the wanted tensors -> (flat, coarse struct or None, fine struct or None,
    latent view or None, (poses, focal, c) views or None)."""
    trainable, (lat, _, cam) = pattern
    case, d_h = st.case, st.case["cfg"]["d_hidden"]
    state = gu.oracle_state(case)
    V, Cc, Hl, Wl = case["latent"].shape
    items = [("c", k, v.shape) for k, v in case["wc"].items() if trainable("c", k)]
    items += [("f", k, v.shape) for k, v in case["wf"].items() if trainable("f", k)]
    if lat:
        items.append(("lat", "", (V, Hl, Wl, Cc)))
    if cam:
        items += [("cam", k, state[k].shape) for k in ("poses", "focal", "c")]
    flat = torch.zeros(sum(torch.Size(s).numel() for _, _, s in items))
    views, off = {"c": {}, "f": {}, "lat": {}, "cam": {}}, 0
    for grp, k, s in items:
        n = torch.Size(s).numel()
        views[grp][k] = flat[off:off + n].view(s)
        off += n

    def struct(sd, g):
        if not g:
            return None
        mm = eu.mlp_struct({k: g.get(k, sd[k]) for k in sd}, d_h)
        for k in sd:
            if k not in g:
                _null(mm, k)
        return mm
    cams = tuple(views["cam"][k] for k in ("poses", "focal", "c")) if cam else None
    return (flat, struct(case["wc"], views["c"]), struct(case["wf"], views["f"]), views["lat"].get(""), cams)


def _cam(cams, keep):
    if cams is None:
        return None
    keep.append(cams)
    return pn.PnrCameraGrad(*(eu.ptr(t) for t in cams))


def _ref(s):
    return C.byref(s) if s is not None else None


def _single_sel(st, a, b, up, pattern):
    keep = []
    flat, gsc, gsf, d_lat, cams = _sel_arena(st, pattern)
    fwd = pn.PnrRenderOut()
    fwd_t = {k: st.rows(st.t[k], a, b) for k in ("z_coarse", "z_fine", "depth_coarse")}
    fwd.z_coarse, fwd.z_fine, fwd.depth_coarse = (eu.ptr(fwd_t["z_coarse"]), eu.ptr(fwd_t["z_fine"]),
                                                  eu.ptr(fwd_t["depth_coarse"]))
    ug = pn.PnrRenderGrad()
    ups = {k: st.rows(v, a, b) for k, v in up.items()}
    for k, v in ups.items():
        setattr(ug, k, eu.ptr(v))
    rays = st.rays[:, a:b].contiguous()
    d_rays = torch.full((st.SB, b - a, 8), float("nan")) if pattern[1][1] else None
    L = eu.lib()
    nbytes = L.pnr_render_backward_workspace_bytes(st.scene, st.mc, st.mf, st.rc, b - a)
    ws = torch.empty(nbytes, dtype=torch.uint8)
    nz = {k: st.rows(v, a, b) for k, v in st.nz.items()}
    eu.ok(L.pnr_render_backward_sel(st.scene, st.mc, st.mf, st.rc, eu.ptr(rays), st.noise(nz), fwd, ug, _ref(gsc),
                                    _ref(gsf), eu.ptr(d_lat), eu.ptr(d_rays), _ref(_cam(cams, keep)), b - a,
                                    ws.data_ptr(), nbytes, None))
    return flat, d_rays


def _sharded_sel(sh, up, pattern):
    st, n, L = sh.st, sh.n, eu.lib()
    want_rays = pattern[1][1]
    keep = []
    sgs = (pn.PnrShardGrad * n)()
    scs = (pn.PnrShardCam * n)()
    flat0, gsc0, gsf0, d_lat0, cam0 = _sel_arena(st, pattern)
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
        flat, gsc, gsf, d_lat, cams = _sel_arena(st, pattern)
        flat.fill_(float("nan"))                        # the driver zeroes the shards' arenas
        sg.grad_coarse = C.pointer(gsc) if gsc is not None else None
        sg.grad_fine = C.pointer(gsf) if gsf is not None else None
        sg.d_latent_nhwc = eu.ptr(d_lat)
        sg.arena, sg.arena_count = eu.ptr(flat), flat.numel()
        if cams is not None:
            scs[i].cam = _cam(cams, keep)
        if not L.pnr_mgpu_peer_load(sh.h, i) and flat.numel() > 0:
            stage0 = torch.full_like(flat, float("nan"))
            sg.arena_stage0 = eu.ptr(stage0)
            keep.append(stage0)
        keep += [flat, gsc, gsf]
    ug = pn.PnrRenderGrad()
    for k, v in up.items():
        setattr(ug, k, eu.ptr(v))
    d_rays0 = torch.full((st.SB, st.B, 8), float("nan")) if want_rays else None
    rc = L.pnr_mgpu_render_backward_sel(sh.h, sh.shards, sgs, scs, st.rc, ug, _ref(gsc0), _ref(gsf0), eu.ptr(d_lat0),
                                        eu.ptr(d_rays0), _ref(_cam(cam0, keep)), st.B, None)
    return rc, flat0, d_rays0


@pytest.mark.parametrize("pattern", ["network_frozen_rays_poses", "coarse_frozen", "blocks_3_4_and_lin_out",
                                     "biases_only"])
@pytest.mark.parametrize("devices", ["peer3", "staged2"])
@pytest.mark.parametrize("name", gu.GRAD_CASE_NAMES)
def test_sharded_sel_equals_separate_sel_calls_summed_in_shard_order(name, devices, pattern):
    import aux_grad_util as au
    st = _Case(name)
    up = au.flat_up(au.load(name), st.R)
    sh = _Sharded(st, DEVICE_LISTS[devices])
    rc, flat, d_rays = _sharded_sel(sh, up, PATTERNS[pattern])
    eu.ok(rc)
    sh.close()
    total, parts = None, []
    for a, b in sh.bounds:
        if b - a <= 0:
            continue
        f, dr = _single_sel(st, a, b, up, PATTERNS[pattern])
        total = f if total is None else total + f
        parts.append(dr)
    assert torch.equal(flat, total)
    if d_rays is not None:
        assert torch.equal(d_rays, torch.cat(parts, dim=1))


def test_sharded_sel_rejects_structs_null_in_other_places():
    import aux_grad_util as au
    st = _Case("sb2_d")
    up = au.flat_up(au.load("sb2_d"), st.R)
    sh = _Sharded(st, [0, 1])
    L = eu.lib()
    pattern = PATTERNS["coarse_frozen"]
    flat0, gsc0, gsf0, d_lat0, _ = _sel_arena(st, pattern)
    flat1, _, gsf1, d_lat1, _ = _sel_arena(st, pattern)
    _, gsc_all, _, _, _ = _sel_arena(st, ALL)
    sgs = (pn.PnrShardGrad * 2)()
    keep = []
    for i, (a, b) in enumerate(sh.bounds):
        t, _ = sh.stage[i]
        sg = sgs[i]
        rays_i = sh.shard_rays(i).contiguous()
        sg.rays, sg.z_coarse, sg.z_fine, sg.depth_coarse = (eu.ptr(rays_i), eu.ptr(t["z_coarse"]),
                                                            eu.ptr(t["z_fine"]), eu.ptr(t["depth_coarse"]))
        up_stage = torch.zeros(st.SB * (b - a) * (8 + 2 * st.Kc + st.Kf))
        ws = torch.empty(L.pnr_render_backward_workspace_bytes(st.scene, st.mc, st.mf, st.rc, b - a),
                         dtype=torch.uint8)
        sg.up_stage, sg.workspace, sg.workspace_bytes = eu.ptr(up_stage), ws.data_ptr(), ws.numel()
        keep += [rays_i, up_stage, ws]
    sgs[0].arena, sgs[0].arena_count = eu.ptr(flat0), flat0.numel()
    sgs[1].arena, sgs[1].arena_count = eu.ptr(flat1), flat1.numel()
    sgs[1].grad_coarse, sgs[1].grad_fine = C.pointer(gsc_all), C.pointer(gsf1)   # device 0's coarse struct is NULL
    sgs[1].d_latent_nhwc = eu.ptr(d_lat1)
    ug = pn.PnrRenderGrad()
    for k, v in up.items():
        setattr(ug, k, eu.ptr(v))
    rc = L.pnr_mgpu_render_backward_sel(sh.h, sh.shards, sgs, None, st.rc, ug, None, _ref(gsf0), eu.ptr(d_lat0), None,
                                        None, st.B, None)
    sh.close()
    assert rc != 0 and b"NULL where" in L.pnr_last_error()
