"""TEST INFRASTRUCTURE: a golden case set up for pnr_render / pnr_render_backward_cam on the host emulator
(tests/cuda_emu), shared by the emulator gradient tests."""
import copy
import ctypes as C

import torch

import emu_util as eu
import golden_util as gu

pn = eu.pn


def case_with_state(name, n_fine=None, n_fine_depth=None, depth_std=0.01, per_object_c=False, seed=0):
    case = copy.copy(gu.load_case(name))
    cfg = dict(case["cfg"], depth_std=depth_std)
    if n_fine is not None:
        cfg.update(n_fine=n_fine, n_fine_depth=n_fine_depth)
        R = cfg["SB"] * cfg["B"]
        case["noise"] = gu.synth.draw_noise(77 + seed, R, cfg["n_coarse"], n_fine, n_fine_depth)
    case["cfg"] = cfg
    st = gu.oracle_state(case)
    if per_object_c:
        g = torch.Generator().manual_seed(seed)
        st["c"] = (st["c"].expand(cfg["SB"], 2) + torch.rand(cfg["SB"], 2, generator=g)).contiguous()
    case["state"] = st
    return case


class Render:
    """pnr_render (SIMT) of a case on the emulator, keeping what the backward needs."""

    def __init__(self, case):
        cfg = case["cfg"]
        self.case, self.keep = case, []
        self.scene = eu.scene_struct(case, case["state"], self.keep)
        self.mc = eu.mlp_struct(case["wc"], cfg["d_hidden"])
        self.mf = eu.mlp_struct(case["wf"], cfg["d_hidden"]) if case["wf"] is not None else None
        self.R, Kc, Kf, Kfd = cfg["SB"] * cfg["B"], cfg["n_coarse"], cfg["n_fine"], cfg["n_fine_depth"]
        rc = pn.PnrRenderCfg()
        rc.n_coarse, rc.n_fine, rc.n_fine_depth, rc.depth_std = Kc, Kf, Kfd, cfg["depth_std"]
        rc.white_bkgd, rc.engine = int(bool(cfg["white_bkgd"])), 1
        self.rc = rc
        self.nz = {k: v.contiguous() for k, v in case["noise"].items()}
        self.lin = torch.linspace(0, 1 - 1.0 / Kc, Kc)
        noise = pn.PnrNoise()
        noise.lin_steps, noise.u_coarse = eu.ptr(self.lin), eu.ptr(self.nz["u_coarse"])
        if Kf - Kfd > 0:
            noise.u_fine, noise.u_fine_jit = eu.ptr(self.nz["u_fine"]), eu.ptr(self.nz["u_fine_jit"])
        if Kf > 0 and Kfd > 0:
            noise.n_depth = eu.ptr(self.nz["n_depth"])
        self.noise = noise
        R = self.R
        t = dict(rgb_coarse=torch.empty(R, 3), depth_coarse=torch.empty(R), weights_coarse=torch.empty(R, Kc),
                 z_coarse=torch.empty(R, Kc))
        if Kf > 0:
            t.update(rgb_fine=torch.empty(R, 3), depth_fine=torch.empty(R), weights_fine=torch.empty(R, Kc + Kf),
                     z_fine=torch.empty(R, Kc + Kf))
        self.out = pn.PnrRenderOut()
        for k, v in t.items():
            setattr(self.out, k, eu.ptr(v))
        self.t = t
        self.rays = case["rays"].contiguous()
        L = eu.lib()
        nbytes = L.pnr_render_workspace_bytes(self.scene, self.mc, self.mf, rc, cfg["B"])
        ws = torch.empty(nbytes, dtype=torch.uint8)
        eu.ok(L.pnr_render(self.scene, self.mc, self.mf, rc, eu.ptr(self.rays), noise, self.out, cfg["B"],
                           ws.data_ptr(), nbytes, None))

    def backward(self, up, rays=False, cam=False, entry="cam"):
        """-> dict(gc, gf, lat, rays, poses, focal, c, launches); up: PnrRenderGrad keys -> tensors."""
        cfg, case, st = self.case["cfg"], self.case, self.case["state"]
        g_c = {k: torch.zeros_like(v) for k, v in case["wc"].items()}
        g_f = {k: torch.zeros_like(v) for k, v in case["wf"].items()} if case["wf"] is not None else None
        gsc = eu.mlp_struct(g_c, cfg["d_hidden"])
        gsf = eu.mlp_struct(g_f, cfg["d_hidden"]) if g_f is not None else None
        V, Cc, Hl, Wl = case["latent"].shape
        d_lat = torch.zeros(V, Hl, Wl, Cc)
        L = eu.lib()
        nbytes = L.pnr_render_backward_workspace_bytes(self.scene, self.mc, self.mf, self.rc, cfg["B"])
        ws = torch.empty(nbytes, dtype=torch.uint8)
        ug = pn.PnrRenderGrad()
        up = {k: v.contiguous() for k, v in up.items() if v is not None}
        for k, v in up.items():
            setattr(ug, k, eu.ptr(v))
        out = dict(gc=g_c, gf=g_f)
        d_rays = torch.full((self.R, 8), float("nan")) if rays else None
        cg = None
        if cam:
            out.update(poses=torch.zeros_like(st["poses"]), focal=torch.zeros_like(st["focal"]),
                       c=torch.zeros_like(st["c"]))
            cg = pn.PnrCameraGrad(eu.ptr(out["poses"]), eu.ptr(out["focal"]), eu.ptr(out["c"]))
        n0 = L.pnr_launch_count()
        if entry == "ex":
            eu.ok(L.pnr_render_backward_ex(self.scene, self.mc, self.mf, self.rc, eu.ptr(self.rays), self.noise,
                                           self.out, ug, gsc, gsf, eu.ptr(d_lat), cfg["B"], ws.data_ptr(), nbytes,
                                           None))
        else:
            eu.ok(L.pnr_render_backward_cam(self.scene, self.mc, self.mf, self.rc, eu.ptr(self.rays), self.noise,
                                            self.out, ug, gsc, gsf, eu.ptr(d_lat), eu.ptr(d_rays),
                                            C.byref(cg) if cg is not None else None, cfg["B"], ws.data_ptr(),
                                            nbytes, None))
        out.update(lat=d_lat, rays=d_rays, launches=L.pnr_launch_count() - n0)
        return out
