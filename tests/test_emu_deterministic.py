"""Deterministic mode on the host emulator (tests/determ_emu.py): the fixed-point latent scatter of the field backward
and the gather-form upsample backward, against oracle/pnr_determinism.py, against the default path and against torch."""
import copy
import ctypes as C
import os
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import determ_emu
import emu_util as eu
import golden_util as gu

sys.path.insert(0, os.path.join(eu.ROOT, "oracle"))
import pnr_determinism as od  # noqa: E402

pn = eu.pn


def rel(a, b):
    return float((a - b).abs().max() / b.abs().max().clamp_min(1e-30))


def _case(name):
    case = copy.copy(gu.load_case(name))
    case["state"] = gu.oracle_state(case)
    return case


def _inputs(case, P, seed, clamp=False):
    cfg = case["cfg"]
    g = torch.Generator().manual_seed(seed)
    rays = case["rays"].reshape(cfg["SB"], -1, 8)
    idx = torch.randint(0, rays.shape[1], (P,), generator=g)
    r = rays[:, idx]
    z = 0.8 + torch.rand(cfg["SB"], P, 1, generator=g)
    xyz = r[..., :3] + z * r[..., 3:6]
    if clamp:          # far outside every view: every point clamps onto the border
        xyz = xyz + torch.tensor([1e3, 1e3, 0.0])
    d_out = torch.randn(cfg["SB"], P, 4, generator=g) * 1e-2
    return xyz.contiguous(), r[..., 3:6].contiguous(), d_out.contiguous()


def _field(L, case, xyz, dirs, d_out, det):
    """pnr_field_backward_cam with every gradient requested, deterministic mode `det` -> dict of outputs."""
    cfg, st = case["cfg"], case["state"]
    keep = []
    scene = eu.scene_struct(case, st, keep)
    wc = case["wc"]
    m = eu.mlp_struct(wc, cfg["d_hidden"])
    g = {k: torch.zeros_like(v) for k, v in wc.items()}
    gs = eu.mlp_struct(g, cfg["d_hidden"])
    SB, P, _ = xyz.shape
    prev = L.pnr_set_deterministic(1 if det else 0)
    try:
        nbytes = L.pnr_field_backward_workspace_bytes(scene, m, P)
        ws = torch.empty(nbytes, dtype=torch.uint8)
        V, Cc, Hl, Wl = case["latent"].shape
        out = dict(g=g, lat=torch.zeros(V, Hl, Wl, Cc), xyz=torch.empty(SB, P, 3), dirs=torch.empty(SB, P, 3),
                   poses=torch.zeros_like(st["poses"]), focal=torch.zeros_like(st["focal"]), c=torch.zeros_like(st["c"]))
        cg = pn.PnrCameraGrad(eu.ptr(out["poses"]), eu.ptr(out["focal"]), eu.ptr(out["c"]))
        rc = L.pnr_field_backward_cam(scene, m, eu.ptr(xyz), eu.ptr(dirs), eu.ptr(d_out), gs, eu.ptr(out["lat"]),
                                       eu.ptr(out["xyz"]), eu.ptr(out["dirs"]), C.byref(cg), P, ws.data_ptr(), nbytes,
                                       None)
        assert rc == 0, L.pnr_last_error().decode()
    finally:
        L.pnr_set_deterministic(prev)
    return out, nbytes


def _oracle_replay(case, xyz, chunks):
    """d_latent of oracle/pnr_determinism.py: every chunk the kernel's scatter received (g0, n, d_lat rows), its taps
    from od.bwd_taps, summed by od.scatter_fixed in chunk order."""
    cfg, st = case["cfg"], case["state"]
    V, Cc, Hl, Wl = case["latent"].shape
    keep = []
    sc = eu.scene_struct(case, st, keep)
    poses = st["poses"].reshape(-1, 12).numpy()
    focal, c = st["focal"].reshape(-1, 2).numpy(), st["c"].reshape(-1, 2).numpy()
    NS, P = cfg["NS"], xyz.shape[1]
    pts = xyz.reshape(-1, 3).numpy()
    out = np.zeros(V * Hl * Wl * Cc, dtype=np.float32)
    for g0, n, d_lat in chunks:
        taps = []
        for lp in range(n):
            g = g0 + lp
            for v in range(NS):
                for off, w in od.bwd_taps(poses, focal, c, NS, Hl, Wl, Cc, (sc.scale_x, sc.scale_y),
                                          (sc.image_w, sc.image_h), g // P, v, pts[g]):
                    taps.append((lp * NS + v, off, w))
        od.scatter_fixed(out, d_lat.reshape(n * NS, Cc), taps, n * NS)
    return out.reshape(V, Hl, Wl, Cc)


def _field_recorded(case, xyz, dirs, d_out):
    """The flag-on field backward with the chunks its fixed-point scatter received -> (outputs, chunks)."""
    chunks = []
    cb = determ_emu.set_chunk_hook(lambda g0, n, d_lat: chunks.append((g0, n, d_lat)))
    try:
        on, _ = _field(determ_emu.lib(), case, xyz, dirs, d_out, True)
    finally:
        determ_emu.set_chunk_hook(None)
    del cb
    return on, chunks


def _assert_same_bits(got, ref):
    got, ref = got.numpy(), np.asarray(ref)
    nan = np.isnan(ref)
    assert np.array_equal(np.isnan(got), nan)
    assert np.array_equal(got[~nan].view(np.uint32), ref[~nan].view(np.uint32))


def _same_except_latent(a, b):
    for k in ("xyz", "dirs", "poses", "focal", "c"):
        assert torch.equal(a[k], b[k]), k
    for k in a["g"]:
        assert torch.equal(a["g"][k], b["g"][k]), k


CASES = [("tiny", None), ("tiny_sb2", None), ("sb2_d", None), ("sb2_d", "10"), ("sb2_d", "21"), ("c3_small", None),
         ("c3_small", "16"), ("c4_small", None), ("c4_small", "20")]   # NS = 2, 1, 3; two objects: sb2_d


@pytest.mark.parametrize("name,chunk_rows", CASES)
def test_fixed_point_latent_gradient(name, chunk_rows, monkeypatch):
    """Flag on: d_latent bit-equal to oracle/pnr_determinism.py replaying the chunks the scatter received, and within
    1e-6 of the float-atomic path (several and ragged chunks with PNR_BWD_CHUNK_ROWS); every other gradient bit-equal
    to the float-atomic path; the workspace query grows."""
    if chunk_rows:
        monkeypatch.setenv("PNR_BWD_CHUNK_ROWS", chunk_rows)
    case = _case(name)
    xyz, dirs, d_out = _inputs(case, 37, 3)
    L = determ_emu.lib()
    off, n_off = _field(L, case, xyz, dirs, d_out, False)
    on, n_on = _field(L, case, xyz, dirs, d_out, True)
    again, _ = _field(L, case, xyz, dirs, d_out, True)
    assert n_on > n_off
    assert float(off["lat"].abs().max()) > 0
    assert rel(on["lat"], off["lat"]) < 1e-6
    _same_except_latent(on, off)
    assert torch.equal(on["lat"], again["lat"])
    _same_except_latent(on, again)
    assert L.pnr_get_deterministic() == 0
    rec, chunks = _field_recorded(case, xyz, dirs, d_out)
    assert len(chunks) == (1 if chunk_rows is None else -(-37 * case["cfg"]["SB"] // (int(chunk_rows) // case["cfg"]["NS"])))
    _assert_same_bits(rec["lat"], _oracle_replay(case, xyz, chunks))


def test_flag_off_is_the_default_library_bit_for_bit():
    case = _case("sb2_d")
    xyz, dirs, d_out = _inputs(case, 37, 5)
    a, na = _field(determ_emu.lib(), case, xyz, dirs, d_out, False)
    b, nb = _field(eu.lib(), case, xyz, dirs, d_out, False)
    assert na == nb
    assert torch.equal(a["lat"], b["lat"])
    _same_except_latent(a, b)


def test_border_pile_up_does_not_overflow():
    """Every point clamps onto the map's border, so a few texels per view take every row's terms: 4 * rows bounds the
    terms per texel, so the int64 sum does not overflow: the result is the oracle's, bit for bit, and within the
    fixed-point bound of the float-atomic sum."""
    case = _case("tiny")
    xyz, dirs, d_out = _inputs(case, 64, 7, clamp=True)
    L = determ_emu.lib()
    on, _ = _field(L, case, xyz, dirs, d_out, True)
    off, _ = _field(L, case, xyz, dirs, d_out, False)
    rec, chunks = _field_recorded(case, xyz, dirs, d_out)
    _assert_same_bits(rec["lat"], _oracle_replay(case, xyz, chunks))
    lat = on["lat"]
    nz = (lat.reshape(-1, lat.shape[-1]).abs().sum(1) > 0).nonzero().flatten()
    assert 1 <= nz.numel() <= 2 * lat.shape[0]
    assert rel(lat, off["lat"]) < 1e-6
    err = (lat.double() - off["lat"].double()).abs().max()
    assert float(err) <= float(off["lat"].abs().max()) * 2.0 ** -20


@pytest.mark.parametrize("bad", [float("nan"), float("inf")])
def test_non_finite_upstream_gradient_reaches_its_taps(bad):
    case = _case("tiny")
    xyz, dirs, d_out = _inputs(case, 16, 9)
    d_out[0, 5, 0] = bad                               # red of one point
    L = determ_emu.lib()
    on, _ = _field(L, case, xyz, dirs, d_out, True)
    off, _ = _field(L, case, xyz, dirs, d_out, False)
    rec, chunks = _field_recorded(case, xyz, dirs, d_out)
    _assert_same_bits(rec["lat"], _oracle_replay(case, xyz, chunks))
    hit = ~torch.isfinite(off["lat"])
    assert hit.any()
    assert not torch.isfinite(on["lat"][hit]).any()
    assert torch.equal(torch.isfinite(on["lat"]), torch.isfinite(off["lat"]))


def test_oracle_scatter_rounding_bound():
    rng = np.random.default_rng(0)
    rows, C, T = 300, 8, 50
    d_lat = (rng.standard_normal((rows, C)) * np.exp(rng.uniform(-20, 5, (rows, 1)))).astype(np.float32)
    taps = [(int(r), int(rng.integers(0, T)) * C, np.float32(rng.uniform(0, 1))) for r in range(rows) for _ in range(4)]
    got = od.scatter_fixed(np.zeros(T * C, dtype=np.float32), d_lat, taps, rows)
    exact = np.zeros(T * C)
    for r, off, w in taps:
        exact[off:off + C] += (d_lat[r] * w).astype(np.float64)
    m = np.abs(d_lat).max()
    e = od.fixed_exponent(m, rows)
    bound = len(taps) * 2.0 ** (-e - 1) + np.abs(exact) * 2.0 ** -24
    assert np.all(np.abs(got - exact) <= bound)
    # the same terms in another order give the same bits
    again = od.scatter_fixed(np.zeros(T * C, dtype=np.float32), d_lat, taps[::-1], rows)
    assert np.array_equal(got.view(np.uint32), again.view(np.uint32))


def _upsample_emu(d_out, h_in, w_in):
    L = determ_emu.lib()
    N, Cc, h_out, w_out = d_out.shape
    d_in = torch.full((N, Cc, h_in, w_in), float("nan"))
    rc = L.pnr_upsample_bilinear_ac_backward(eu.ptr(d_out), N, Cc, h_in, w_in, h_out, w_out, eu.ptr(d_in), None)
    assert rc == 0, L.pnr_last_error().decode()
    return d_in


# the encoder's maps: conv1 / layer1..3 of the C2 and C4 inputs (128 x 128 and 300 x 400 images) onto conv1's size,
# the same-size map, and a size of 1 on either side
SHAPES = [((32, 32), (64, 64)), ((16, 16), (64, 64)), ((8, 8), (64, 64)), ((64, 64), (64, 64)),
          ((75, 100), (150, 200)), ((38, 50), (150, 200)), ((19, 25), (150, 200)), ((150, 200), (150, 200)),
          ((1, 1), (5, 7)), ((1, 4), (6, 9)), ((5, 3), (1, 1)), ((4, 6), (1, 8)), ((3, 1), (7, 1))]


@pytest.mark.parametrize("hw_in,hw_out", SHAPES)
def test_upsample_backward(hw_in, hw_out):
    g = torch.Generator().manual_seed(hw_in[0] * 1000 + hw_out[1])
    d_out = torch.randn(2, 3, *hw_out, generator=g)
    got = _upsample_emu(d_out, *hw_in)
    ref = od.upsample_ac_backward(d_out.numpy(), *hw_in)
    assert np.array_equal(got.numpy().view(np.uint32), ref.view(np.uint32))
    x = torch.randn(2, 3, *hw_in, generator=g, dtype=torch.float64).float().requires_grad_(True)
    F.interpolate(x, hw_out, mode="bilinear", align_corners=True).backward(d_out)
    assert rel(got, x.grad) < 1e-6


def test_upsample_backward_argument_errors():
    L = determ_emu.lib()
    d = torch.zeros(1, 1, 2, 2)
    assert L.pnr_upsample_bilinear_ac_backward(eu.ptr(d), 1, 1, 0, 2, 2, 2, eu.ptr(d), None) == pn_err_invalid()
    assert L.pnr_upsample_bilinear_ac_backward(None, 1, 1, 2, 2, 2, 2, eu.ptr(d), None) == pn_err_invalid()
    assert L.pnr_upsample_bilinear_ac_backward(None, 0, 1, 2, 2, 2, 2, None, None) == 0


def pn_err_invalid():
    import re
    h = open(os.path.join(eu.ROOT, "include", "pnr.h")).read()
    return int(re.search(r"PNR_ERR_INVALID\s*=?\s*\(?(-?\d+)", h).group(1))
