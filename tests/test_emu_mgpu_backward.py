"""pnr_mgpu_render_backward (csrc/pnr_mgpu.cu: the backward of the ray-sharded render behind `bind_parallel(net, gpus)`
in grad mode) and its reduction pnr_sum_into on the host emulator.  The emulator has one device; device lists with
distinct ids take the peer-read path of the reduction, repeated ids the staged one (device 0 cannot address "itself"
as a peer).  The driver's gradients must equal, bit for bit, n separate pnr_render_backward_ex calls over the same
slices summed in shard order, and agree with one call over all rays up to summation order."""
import ctypes as C

import pytest
import torch

import aux_grad_util as au
import emu_util as eu
import golden_util as gu

pn = eu.pn
rel = au.rel

DEVICE_LISTS = {"peer3": [0, 1, 2],          # distinct devices: the reduction reads each arena in place
                "staged2": [0, 0],           # no peer access: the arena is copied to device 0 first
                "eight": list(range(8)),     # sb2_d (B = 12): shards 6 and 7 get no rays
                "sb_pair": [0, 1]}


class _Case:
    """A golden case on the emulator: scene, MLPs, config and draws, plus one forward over all rays."""

    def __init__(self, name):
        case = gu.load_case(name)
        cfg = case["cfg"]
        self.case, self.keep = case, []
        self.SB, self.B = cfg["SB"], cfg["B"]
        self.Kc, self.Kf, self.Kfd = cfg["n_coarse"], cfg["n_fine"], cfg["n_fine_depth"]
        self.R = self.SB * self.B
        self.scene = eu.scene_struct(case, gu.oracle_state(case), self.keep)
        self.mc = eu.mlp_struct(case["wc"], cfg["d_hidden"])
        self.mf = eu.mlp_struct(case["wf"], cfg["d_hidden"])
        rc = pn.PnrRenderCfg()
        rc.n_coarse, rc.n_fine, rc.n_fine_depth, rc.depth_std = self.Kc, self.Kf, self.Kfd, 0.01
        rc.white_bkgd, rc.engine = int(bool(cfg["white_bkgd"])), 1
        self.rc = rc
        self.rays = case["rays"].contiguous()
        self.nz = {k: v.contiguous() for k, v in case["noise"].items()}
        self.lin = torch.linspace(0, 1 - 1.0 / self.Kc, self.Kc)
        self.t, self.out = self.outputs(self.R)
        L = eu.lib()
        nbytes = L.pnr_render_workspace_bytes(self.scene, self.mc, self.mf, rc, self.B)
        ws = torch.empty(nbytes, dtype=torch.uint8)
        eu.ok(L.pnr_render(self.scene, self.mc, self.mf, rc, eu.ptr(self.rays), self.noise(self.nz), self.out, self.B,
                           ws.data_ptr(), nbytes, None))

    def noise(self, nz):
        noise = pn.PnrNoise()
        noise.lin_steps, noise.u_coarse = eu.ptr(self.lin), eu.ptr(nz["u_coarse"])
        if self.Kf - self.Kfd > 0:
            noise.u_fine, noise.u_fine_jit = eu.ptr(nz["u_fine"]), eu.ptr(nz["u_fine_jit"])
        if self.Kfd > 0:
            noise.n_depth = eu.ptr(nz["n_depth"])
        self.keep.append(nz)
        return noise

    def outputs(self, R):
        K = self.Kc + self.Kf
        t = dict(rgb_coarse=torch.full((R, 3), -7.0), depth_coarse=torch.full((R,), -7.0),
                 z_coarse=torch.full((R, self.Kc), -7.0), rgb_fine=torch.full((R, 3), -7.0),
                 depth_fine=torch.full((R,), -7.0), z_fine=torch.full((R, K), -7.0))
        o = pn.PnrRenderOut()
        for k, v in t.items():
            setattr(o, k, eu.ptr(v))
        return t, o

    def rows(self, x, a, b):
        """Rays [a, b) of every object of a per-ray tensor [SB*B][...] -> [SB*(b-a)][...] (1-D stays 1-D)."""
        y = x.reshape(self.SB, self.B, -1)[:, a:b]
        return y.reshape(-1).contiguous() if x.dim() == 1 else y.reshape(self.SB * (b - a), -1).contiguous()

    def arena(self, want_latent=True):
        """One flat gradient buffer holding both MLPs' parameter gradients and the NHWC latent gradient ->
        (flat, coarse dict, fine dict, latent view or None, coarse struct, fine struct)."""
        case, d_h = self.case, self.case["cfg"]["d_hidden"]
        V, Cc, Hl, Wl = case["latent"].shape
        shapes = [("c", k, v.shape) for k, v in case["wc"].items()] + [("f", k, v.shape) for k, v in case["wf"].items()]
        if want_latent:
            shapes.append(("lat", "", (V, Hl, Wl, Cc)))
        flat = torch.zeros(sum(torch.Size(s).numel() for _, _, s in shapes))
        views, off = {"c": {}, "f": {}, "lat": {}}, 0
        for grp, k, s in shapes:
            n = torch.Size(s).numel()
            views[grp][k] = flat[off:off + n].view(s)
            off += n
        return (flat, views["c"], views["f"], views["lat"].get(""), eu.mlp_struct(views["c"], d_h),
                eu.mlp_struct(views["f"], d_h))

    def backward(self, rays, nz, fwd_t, up, B, want_latent=True):
        """One pnr_render_backward_ex into a fresh zeroed arena -> (flat, coarse, fine, latent)."""
        flat, g_c, g_f, d_lat, gsc, gsf = self.arena(want_latent)
        fwd = pn.PnrRenderOut()
        fwd.z_coarse, fwd.z_fine, fwd.depth_coarse = (eu.ptr(fwd_t["z_coarse"]), eu.ptr(fwd_t["z_fine"]),
                                                      eu.ptr(fwd_t["depth_coarse"]))
        ug = pn.PnrRenderGrad()
        for k, v in up.items():
            setattr(ug, k, eu.ptr(v))
        L = eu.lib()
        nbytes = L.pnr_render_backward_workspace_bytes(self.scene, self.mc, self.mf, self.rc, B)
        ws = torch.empty(nbytes, dtype=torch.uint8)
        eu.ok(L.pnr_render_backward_ex(self.scene, self.mc, self.mf, self.rc, eu.ptr(rays), self.noise(nz), fwd, ug,
                                       gsc, gsf, eu.ptr(d_lat), B, ws.data_ptr(), nbytes, None))
        return flat, g_c, g_f, d_lat


def _upstream(st, name, mode):
    """rgb: the MSE gradients of train.py's loss against the grad_* fixture's target; all: grad_aux_*'s six."""
    if mode == "rgb":
        gt = gu.load_grad_case(name)["rgb_gt"].reshape(st.R, 3).float()
        return {k: (2.0 * (st.t[k.replace("d_", "")] - gt) / gt.numel()).contiguous()
                for k in ("d_rgb_coarse", "d_rgb_fine")}
    return au.flat_up(au.load(name), st.R)


class _Sharded:
    """The forward and backward of one case through the multi-GPU driver on `devices`."""

    def __init__(self, st, devices):
        self.st, self.devices = st, devices
        self.n = n = len(devices)
        L = eu.lib()
        self.h = C.c_void_p()
        eu.ok(L.pnr_mgpu_create((C.c_int32 * n)(*devices), n, C.byref(self.h)))
        self.shards = (pn.PnrShard * n)()
        self.stage = {}
        self.keep = []
        per = -(-st.B // n)
        self.bounds = [(min(st.B, per * i), min(st.B, per * (i + 1))) for i in range(n)]
        for i, (a, b) in enumerate(self.bounds):
            Bi = b - a
            if Bi <= 0:
                continue
            sub = {k: st.rows(v, a, b) for k, v in st.nz.items()}
            t, o = st.outputs(st.SB * Bi)
            wsb = L.pnr_render_workspace_bytes(st.scene, st.mc, st.mf, st.rc, Bi)
            ws = torch.empty(wsb, dtype=torch.uint8)
            rays_stage = torch.full((st.SB, Bi, 8), float("nan"))
            sh = self.shards[i]
            sh.scene, sh.mlp_coarse, sh.mlp_fine = C.pointer(st.scene), C.pointer(st.mc), C.pointer(st.mf)
            sh.noise = C.pointer(st.noise(sub))
            sh.workspace, sh.workspace_bytes = ws.data_ptr(), wsb
            sh.rays_stage = eu.ptr(rays_stage)
            sh.stage = o
            self.stage[i] = (t, rays_stage)
            self.keep += [ws, sh.noise]
        # the forward: out0 asks for no sample depths, the stages keep them for the backward
        self.t0, o0 = st.outputs(st.R)
        o0.z_coarse = o0.z_fine = None
        eu.ok(L.pnr_mgpu_render(self.h, self.shards, st.rc, eu.ptr(st.rays), o0, st.B, None))

    def shard_rays(self, i):
        a, b = self.bounds[i]
        if i == 0 and self.st.SB == 1:
            return self.st.rays[:, a:b]          # shard 0 of one object renders in place from device 0's rays
        return self.stage[i][1]

    def backward(self, up, want_latent=True, break_shard=None):
        st, n, L = self.st, self.n, eu.lib()
        K = st.Kc + st.Kf
        sgs = (pn.PnrShardGrad * n)()
        flat0, g_c0, g_f0, d_lat0, gsc0, gsf0 = st.arena(want_latent)
        for i, (a, b) in enumerate(self.bounds):
            Bi = b - a
            if Bi <= 0:
                continue
            t, _ = self.stage[i]
            sg = sgs[i]
            rays_i = self.shard_rays(i).contiguous()
            sg.rays, sg.z_coarse, sg.z_fine, sg.depth_coarse = (eu.ptr(rays_i), eu.ptr(t["z_coarse"]),
                                                                eu.ptr(t["z_fine"]), eu.ptr(t["depth_coarse"]))
            up_stage = torch.full((st.SB * Bi * (8 + 2 * st.Kc + st.Kf),), float("nan"))
            sg.up_stage = eu.ptr(up_stage)
            wsb = L.pnr_render_backward_workspace_bytes(st.scene, st.mc, st.mf, st.rc, Bi)
            ws = torch.empty(wsb, dtype=torch.uint8)
            sg.workspace, sg.workspace_bytes = ws.data_ptr(), wsb
            self.keep += [rays_i, up_stage, ws]
            if i == 0:
                sg.arena, sg.arena_count = eu.ptr(flat0), flat0.numel()
                continue
            flat, _, _, d_lat, gsc, gsf = st.arena(want_latent)
            flat.fill_(float("nan"))                        # the driver zeroes the shards' arenas
            sg.grad_coarse, sg.grad_fine, sg.d_latent_nhwc = C.pointer(gsc), C.pointer(gsf), eu.ptr(d_lat)
            sg.arena, sg.arena_count = eu.ptr(flat), flat.numel()
            if not L.pnr_mgpu_peer_load(self.h, i):
                stage0 = torch.full_like(flat, float("nan"))
                sg.arena_stage0 = eu.ptr(stage0)
                self.keep.append(stage0)
            self.keep += [flat, gsc, gsf]
        if break_shard is not None:
            break_shard(sgs)
        ug = pn.PnrRenderGrad()
        for k, v in up.items():
            setattr(ug, k, eu.ptr(v))
        rc = L.pnr_mgpu_render_backward(self.h, self.shards, sgs, st.rc, ug, gsc0, gsf0, eu.ptr(d_lat0), st.B, None)
        return rc, (flat0, g_c0, g_f0, d_lat0)

    def close(self):
        eu.ok(eu.lib().pnr_mgpu_destroy(self.h))


@pytest.mark.parametrize("mode", ["rgb", "all"])
@pytest.mark.parametrize("devices", list(DEVICE_LISTS))
@pytest.mark.parametrize("name", gu.GRAD_CASE_NAMES)
def test_sharded_backward_equals_separate_calls_summed_in_shard_order(name, devices, mode):
    st = _Case(name)
    up = _upstream(st, name, mode)
    sh = _Sharded(st, DEVICE_LISTS[devices])
    for k in ("rgb_coarse", "depth_coarse", "rgb_fine", "depth_fine"):
        assert torch.equal(sh.t0[k], st.t[k]), k
    assert torch.equal(sh.t0["z_coarse"], torch.full_like(st.t["z_coarse"], -7.0))   # not copied back to device 0
    rc, (flat, g_c, g_f, d_lat) = sh.backward(up)
    eu.ok(rc)
    sh.close()
    # n separate calls over the same slices, summed left to right
    total = None
    for i, (a, b) in enumerate(sh.bounds):
        if b - a <= 0:
            continue
        fwd = {k: st.rows(st.t[k], a, b) for k in ("z_coarse", "z_fine", "depth_coarse")}
        part = st.backward(st.rays[:, a:b].contiguous(), {k: st.rows(v, a, b) for k, v in st.nz.items()}, fwd,
                           {k: st.rows(v, a, b) for k, v in up.items()}, b - a)[0]
        total = part if total is None else total + part
    if devices == "eight" and name == "sb2_d":
        assert sh.bounds[-1][1] - sh.bounds[-1][0] <= 0      # the trailing shards are empty
    assert flat.abs().max() > 0
    assert torch.equal(flat, total)
    # one call over all rays: the same gradients up to the order of summation
    whole, w_c, w_f, w_lat = st.backward(st.rays, st.nz, st.t, up, st.B)
    assert rel(d_lat, w_lat) <= 1e-5
    for k in w_c:
        assert rel(g_c[k], w_c[k]) <= 1e-5, ("coarse", k)
    for k in w_f:
        assert rel(g_f[k], w_f[k]) <= 1e-5, ("fine", k)
    if mode == "all":    # and the reference's own gradients, at the bar the single-call backward meets
        aux = au.load(name)
        assert rel(d_lat.permute(0, 3, 1, 2), aux["g_latent"]) < 5e-4
        for k, v in aux["gc"].items():
            assert rel(g_c[k], v) < 5e-4, ("coarse vs reference", k)


def test_sharded_backward_without_latent_gradient():
    """stop_encoder_grad: no latent gradient anywhere, the arenas hold the parameter gradients only."""
    st = _Case("sb2_d")
    up = _upstream(st, "sb2_d", "all")
    sh = _Sharded(st, [0, 1, 2])
    rc, (flat, _, _, d_lat) = sh.backward(up, want_latent=False)
    eu.ok(rc)
    sh.close()
    whole = st.backward(st.rays, st.nz, st.t, up, st.B, want_latent=False)[0]
    assert d_lat is None
    assert rel(flat, whole) <= 1e-5


@pytest.mark.parametrize("n", [1, 2, 5])
@pytest.mark.parametrize("count", [0, 1, 3, 4, 7, 1025])
@pytest.mark.parametrize("offset", [0, 1, 3])
def test_sum_into_adds_sources_left_to_right(n, count, offset):
    """Ragged counts and pointers off the 16-byte grid (the float4 body is then not taken): bit-equal to adding the
    sources one after another."""
    g = torch.Generator().manual_seed(n * 1000 + count + offset)
    base = [torch.randn(count + offset, generator=g) * 10 ** float(k % 3) for k in range(n + 1)]
    dst = base[0][offset:]
    ref = dst.clone()
    for s in base[1:]:
        ref = ref + s[offset:]
    srcs = (C.c_void_p * max(n, 1))(*[s[offset:].data_ptr() for s in base[1:]])
    eu.ok(eu.lib().pnr_sum_into(C.c_void_p(dst.data_ptr()), srcs, n, count, None))
    assert torch.equal(dst, ref)


def test_sum_into_rejects_bad_arguments():
    L = eu.lib()
    dst = torch.zeros(8)
    srcs = (C.c_void_p * 2)(torch.zeros(8).data_ptr(), None)
    assert L.pnr_sum_into(eu.ptr(dst), srcs, 2, 8, None) < 0
    assert b"NULL source" in L.pnr_last_error()
    assert L.pnr_sum_into(eu.ptr(dst), srcs, 64, 8, None) < 0
    assert L.pnr_sum_into(eu.ptr(dst), srcs, 1, -1, None) < 0


def _clear(field, i=1):
    def br(sgs):
        setattr(sgs[i], field, None)
    return br


@pytest.mark.parametrize("devices,breaker,message", [
    ([0, 1], _clear("z_coarse"), b"incomplete shard gradient"),
    ([0, 1], _clear("up_stage"), b"staging buffer"),
    ([0, 1], _clear("grad_fine"), b"grad_coarse / grad_fine"),
    ([0, 1], _clear("arena", 0), b"device 0's gradient arena"),
    ([0, 0], _clear("arena_stage0"), b"no peer access"),
    ([0, 1], lambda sgs: setattr(sgs[1], "arena_count", sgs[1].arena_count - 1), b"arena of device 0's size"),
    ([0, 1], lambda sgs: setattr(sgs[1], "d_latent_nhwc", sgs[1].d_latent_nhwc + 4), b"layout"),
])
def test_sharded_backward_rejects_incomplete_structs(devices, breaker, message):
    st = _Case("sb2_d")
    sh = _Sharded(st, devices)
    rc, _ = sh.backward(_upstream(st, "sb2_d", "all"), break_shard=breaker)
    sh.close()
    assert rc < 0
    assert message in eu.lib().pnr_last_error()


def test_sharded_backward_rejects_missing_arguments():
    st = _Case("tiny")
    sh = _Sharded(st, [0, 1])
    L = eu.lib()
    sgs = (pn.PnrShardGrad * 2)()
    assert L.pnr_mgpu_render_backward(sh.h, sh.shards, sgs, st.rc, None, None, None, None, st.B, None) < 0
    assert b"NULL argument" in L.pnr_last_error()
    assert L.pnr_mgpu_render_backward(sh.h, sh.shards, sgs, st.rc, None, st.mc, st.mf, None, st.B, None) < 0
    assert b"shard gradient" in L.pnr_last_error()
    sh.close()
