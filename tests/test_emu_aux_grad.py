"""Gradients of the depth and weights outputs through the C ABI, CUDA sources executed on the CPU by the host emulator
of tests/cuda_emu: `pnr_composite_backward` against the oracle's compositing backward, and `pnr_render_backward_ex`
against the oracle's render_backward and the reference's own gradients for a loss on all six outputs."""
import copy
import os

import pytest
import torch

import aux_grad_util as au
import emu_util as eu
import golden_util as gu

ab = gu.load_by_path("pnr_aux_backward", os.path.join(gu.ROOT, "oracle", "pnr_aux_backward.py"))
rel = au.rel


@pytest.mark.parametrize("K", [1, 2, 9])
@pytest.mark.parametrize("white", [0, 1])
@pytest.mark.parametrize("with_rgb,with_depth,with_weights", [(1, 1, 1), (0, 0, 1), (1, 0, 0), (0, 1, 0)])
def test_composite_backward_matches_oracle(K, white, with_rgb, with_depth, with_weights):
    """Random rays / sorted depths / field values with a quarter of the sigmas <= 0 (no density gradient there)."""
    g = torch.Generator().manual_seed(100 * K + 10 * white + 4 * with_rgb + 2 * with_depth + with_weights)
    R = 37
    rays = torch.zeros(R, 8)
    rays[:, 3:6] = torch.nn.functional.normalize(torch.randn(R, 3, generator=g), dim=-1)
    rays[:, 6], rays[:, 7] = 0.8, 1.8
    z = torch.sort(0.8 + torch.rand(R, K, generator=g), dim=-1)[0].contiguous()
    field = torch.cat((torch.rand(R, K, 3, generator=g), torch.randn(R, K, 1, generator=g) * 3.0), -1)
    field[..., 3][torch.rand(R, K, generator=g) < 0.25] = 0.0
    field = field.contiguous()
    d_rgb = torch.randn(R, 3, generator=g) if with_rgb else None
    d_depth = torch.randn(R, generator=g) if with_depth else None
    d_w = torch.randn(R, K, generator=g) if with_weights else None
    ref_field, ref_z = ab.composite_backward(rays, z, field, d_rgb, d_depth, d_w, bool(white))
    d_field, d_z = torch.full((R, K, 4), float("nan")), torch.full((R, K), float("nan"))
    eu.ok(eu.lib().pnr_composite_backward(eu.ptr(rays), eu.ptr(z), eu.ptr(field), white, eu.ptr(d_rgb),
                                          eu.ptr(d_depth), eu.ptr(d_w), eu.ptr(d_field), eu.ptr(d_z), R, K, None))
    assert ref_field.abs().max() > 0
    assert rel(d_field, ref_field) < 1e-5
    assert rel(d_z, ref_z) < 1e-5
    assert torch.all(d_field[..., 3][field[..., 3] <= 0] == 0)


class _Step:
    """pnr_render (SIMT) of a golden case on the emulator, keeping what pnr_render_backward(_ex) needs."""

    def __init__(self, case):
        pn = eu.pn
        cfg = case["cfg"]
        self.case, self.keep = case, []
        self.scene = eu.scene_struct(case, gu.oracle_state(case), self.keep)
        self.mc = eu.mlp_struct(case["wc"], cfg["d_hidden"])
        self.mf = eu.mlp_struct(case["wf"], cfg["d_hidden"]) if case["wf"] is not None else None
        self.R, Kc, Kf, Kfd = cfg["SB"] * cfg["B"], cfg["n_coarse"], cfg["n_fine"], cfg["n_fine_depth"]
        rc = pn.PnrRenderCfg()
        rc.n_coarse, rc.n_fine, rc.n_fine_depth, rc.depth_std = Kc, Kf, Kfd, 0.01
        rc.white_bkgd, rc.engine = int(bool(cfg["white_bkgd"])), 1
        self.rc = rc
        nz = {k: v.contiguous() for k, v in case["noise"].items()}
        self.lin = torch.linspace(0, 1 - 1.0 / Kc, Kc)
        noise = pn.PnrNoise()
        noise.lin_steps, noise.u_coarse = eu.ptr(self.lin), eu.ptr(nz["u_coarse"])
        if Kf - Kfd > 0:
            noise.u_fine, noise.u_fine_jit = eu.ptr(nz["u_fine"]), eu.ptr(nz["u_fine_jit"])
        if Kfd > 0:
            noise.n_depth = eu.ptr(nz["n_depth"])
        self.nz, self.noise = nz, noise
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

    def backward(self, up=None, rgb_only_entry=False):
        """-> (grads_coarse, grads_fine or None, d_latent NCHW).  up: PnrRenderGrad keys -> tensors (None = NULL)."""
        cfg, case = self.case["cfg"], self.case
        g_c = {k: torch.zeros_like(v) for k, v in case["wc"].items()}
        g_f = {k: torch.zeros_like(v) for k, v in case["wf"].items()} if case["wf"] is not None else None
        gsc = eu.mlp_struct(g_c, cfg["d_hidden"])
        gsf = eu.mlp_struct(g_f, cfg["d_hidden"]) if g_f is not None else None
        V, Cc, Hl, Wl = case["latent"].shape
        d_lat = torch.zeros(V, Hl, Wl, Cc)
        L = eu.lib()
        nbytes = L.pnr_render_backward_workspace_bytes(self.scene, self.mc, self.mf, self.rc, cfg["B"])
        ws = torch.empty(nbytes, dtype=torch.uint8)
        up = {k: (v.contiguous() if v is not None else None) for k, v in (up or {}).items()}
        if rgb_only_entry:
            eu.ok(L.pnr_render_backward(self.scene, self.mc, self.mf, self.rc, eu.ptr(self.rays), self.noise, self.out,
                                        eu.ptr(up.get("d_rgb_coarse")), eu.ptr(up.get("d_rgb_fine")), gsc, gsf,
                                        eu.ptr(d_lat), cfg["B"], ws.data_ptr(), nbytes, None))
        else:
            ug = eu.pn.PnrRenderGrad()
            for k, v in up.items():
                setattr(ug, k, eu.ptr(v))
            eu.ok(L.pnr_render_backward_ex(self.scene, self.mc, self.mf, self.rc, eu.ptr(self.rays), self.noise,
                                           self.out, ug, gsc, gsf, eu.ptr(d_lat), cfg["B"], ws.data_ptr(), nbytes,
                                           None))
        return g_c, g_f, d_lat.permute(0, 3, 1, 2)


def _oracle(case, up):
    cfg = case["cfg"]
    return ab.render_backward(case["rays"], case["noise"], gu.oracle_state(case), case["latent"], case["wc"],
                              case["wf"], cfg["NS"], cfg["n_coarse"], cfg["n_fine"], cfg["n_fine_depth"], up,
                              white_bkgd=bool(cfg["white_bkgd"]))


def _same_samples(case, step):
    """The comparison needs identical samples: no ray may have flipped a CDF bin."""
    if case["cfg"]["n_fine"] > 0:
        ref = gu.oracle_render(case)
        assert (step.t["z_fine"] - ref["fine"]["z"]).abs().max() < 1e-5


@pytest.mark.parametrize("name", au.CASE_NAMES)
def test_emulated_render_backward_ex_matches_reference_gradients(name):
    case, aux = gu.load_case(name), au.load(name)
    step = _Step(case)
    _same_samples(case, step)
    up = au.flat_up(aux, step.R)
    g_c, g_f, d_lat = step.backward(up)
    o_c, o_f, o_lat = _oracle(case, up)
    assert rel(d_lat, o_lat) < 2e-4
    for k in o_c:
        assert rel(g_c[k], o_c[k]) < 2e-4, ("coarse", k)
    for k in o_f:
        assert rel(g_f[k], o_f[k]) < 2e-4, ("fine", k)
    assert rel(d_lat, aux["g_latent"]) < 5e-4
    for k, v in aux["gc"].items():
        assert rel(g_c[k], v) < 5e-4, ("coarse vs reference", k)
    for k, v in aux["gf"].items():
        assert rel(g_f[k], v) < 5e-4, ("fine vs reference", k)


@pytest.mark.parametrize("n_fine,n_fine_depth", [(0, 0), (6, 0), (4, 4), (5, 1)])
def test_emulated_render_backward_ex_sample_count_edge_cases(n_fine, n_fine_depth):
    """Coarse only, no depth-centred samples, only depth-centred samples and a single one: random upstream gradients
    of every output against the oracle with the same noise."""
    case = copy.copy(gu.load_case("sb2_d"))
    cfg = dict(case["cfg"], n_fine=n_fine, n_fine_depth=n_fine_depth)
    case["cfg"] = cfg
    R, Kc = cfg["SB"] * cfg["B"], cfg["n_coarse"]
    case["noise"] = gu.synth.draw_noise(77, R, Kc, n_fine, n_fine_depth)
    g = torch.Generator().manual_seed(n_fine * 10 + n_fine_depth)
    up = dict(d_rgb_coarse=torch.randn(R, 3, generator=g), d_depth_coarse=torch.randn(R, generator=g),
              d_weights_coarse=torch.randn(R, Kc, generator=g))
    if n_fine > 0:
        up.update(d_rgb_fine=torch.randn(R, 3, generator=g), d_depth_fine=torch.randn(R, generator=g),
                  d_weights_fine=torch.randn(R, Kc + n_fine, generator=g))
    up = {k: v * 1e-2 for k, v in up.items()}
    step = _Step(case)
    _same_samples(case, step)
    g_c, g_f, d_lat = step.backward(up)
    o_c, o_f, o_lat = _oracle(case, up)
    assert o_lat.abs().max() > 0
    assert rel(d_lat, o_lat) < 2e-4
    for k in o_c:
        assert rel(g_c[k], o_c[k]) < 2e-4, ("coarse", k)
    for k in (o_f or {}):
        assert rel(g_f[k], o_f[k]) < 2e-4, ("fine", k)


@pytest.mark.parametrize("name", ["sb2_d", "tiny", "ns1_coarse_only"])
def test_emulated_fine_outputs_only_reach_the_coarse_mlp_through_the_depth_samples(name):
    """Gradients on the fine depth / weights alone (no coarse-output gradient): the coarse MLP still receives one
    through the depth-centred samples when there are any, and none when the pass has no fine samples."""
    case = gu.load_case(name)
    cfg = case["cfg"]
    step = _Step(case)
    R, K = step.R, cfg["n_coarse"] + cfg["n_fine"]
    g = torch.Generator().manual_seed(4)
    up = dict(d_depth_fine=torch.randn(R, generator=g), d_weights_fine=torch.randn(R, K, generator=g))
    g_c, g_f, _ = step.backward(up if cfg["n_fine"] > 0 else {})
    reached = g_c["blocks.4.fc_1.weight"].abs().max() > 0
    assert reached == (cfg["n_fine"] > 0 and cfg["n_fine_depth"] > 0)
    if cfg["n_fine"] > 0:
        o_c, o_f, _ = _oracle(case, up)
        for k in o_c:
            assert rel(g_c[k], o_c[k]) < 2e-4, ("coarse", k)


@pytest.mark.parametrize("name", gu.GRAD_CASE_NAMES + ["ns1_coarse_only"])
def test_rgb_only_entry_point_equals_ex_with_null_aux_gradients(name):
    """pnr_render_backward is pnr_render_backward_ex with NULL depth / weights gradients, bit for bit."""
    case = gu.load_case(name)
    cfg = case["cfg"]
    step = _Step(case)
    g = torch.Generator().manual_seed(8)
    up = dict(d_rgb_coarse=torch.randn(step.R, 3, generator=g) * 1e-2)
    if cfg["n_fine"] > 0:
        up["d_rgb_fine"] = torch.randn(step.R, 3, generator=g) * 1e-2
    a_c, a_f, a_lat = step.backward(up, rgb_only_entry=True)
    b_c, b_f, b_lat = step.backward(up)
    assert a_lat.abs().max() > 0
    assert torch.equal(a_lat, b_lat)
    for k in a_c:
        assert torch.equal(a_c[k], b_c[k]), ("coarse", k)
    for k in (a_f or {}):
        assert torch.equal(a_f[k], b_f[k]), ("fine", k)
