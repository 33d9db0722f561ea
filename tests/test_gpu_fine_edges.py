"""Shapes of the fused render that stress its ray flush (csrc/pnr_field_tc.cu finish_ray), checked on every ray by
tests/fine_pass_check.py: the merged samples bit-equal to the stage kernel and explained by the kernel's own coarse
weights, the fine outputs against the oracle at the kernel's own samples, and the coarse outputs against the oracle
at the kernel's coarse samples.  c2_small's scene and MLPs, fresh noise per shape.

  (8, 8, 4), (20, 12, 4)      n_coarse < 32: idle lanes in the cdf's warp-tree sum
  (33, 31, 0), (100, 28, 28)  n_coarse not a multiple of 32; no importance samples at all
  (200, 100, 20)              300 samples: every ray spans five or more CTAs, K does not divide 64
  (448, 64, 16), (511, 1, 0)  K = 512: the staged flush at its scratch limit
  (512, 0, 0)                 coarse only, 6 Kc + Kc + 1 + K = 4097 floats: the unstaged flush (L2 loads)
and R = 1, R = 3 at (64, 32, 16) (3 fine tiles of 128 points, 2 coarse ones: one CTA pair starts in the fine pass),
two objects with an odd B, a black background, and a depth_std that clamps depth samples to near and to far.
Engines: "tc", "tc_fast" (against tests/tc_fast_oracle.py) and the SIMT engine as a control."""
import pytest

import fine_pass_check as fpc
import golden_util as gu
import gpu_util
import tc_fast_oracle as fo

pytestmark = pytest.mark.gpu

SHAPES = [(8, 8, 4), (20, 12, 4), (33, 31, 0), (100, 28, 28), (200, 100, 20), (448, 64, 16), (511, 1, 0),
          (512, 0, 0)]
# name -> (Kc, Kf, Kfd, R, SB, white_bkgd, depth_std)
CASES = {f"K{Kc}_{Kf}_{Kfd}": (Kc, Kf, Kfd, 24, 1, True, 0.01) for Kc, Kf, Kfd in SHAPES}
CASES.update({
    "R1": (64, 32, 16, 1, 1, True, 0.01),
    "R3": (64, 32, 16, 3, 1, True, 0.01),
    "SB2_B7": (64, 32, 16, 7, 2, True, 0.01),
    "black_bkgd": (64, 32, 16, 24, 1, False, 0.01),
    "depth_clamps": (64, 32, 16, 24, 1, True, 2.0),
})
ENGINES = ["tc", "tc_fast", "simt"]


def _case(name):
    Kc, Kf, Kfd, R, SB, white, depth_std = CASES[name]
    case = dict(gu.load_case("c2_small"))
    cfg = dict(case["cfg"], n_coarse=Kc, n_fine=Kf, n_fine_depth=Kfd, white_bkgd=white, B=R)
    if SB == 2:
        # the two source views become two single-view objects with their own rays (test_gpu_tc.py two_objects)
        case["rays"] = case["rays"][0, :2 * R].reshape(2, R, 8).contiguous()
        case["src_poses"] = case["src_poses"].reshape(2, 1, 4, 4).contiguous()
        cfg.update(SB=2, NS=1)
    else:
        case["rays"] = case["rays"][:, :R].contiguous()
    case["cfg"] = cfg
    case["noise"] = gu.synth.draw_noise(1000 + sorted(CASES).index(name), SB * R, Kc, Kf, Kfd)
    return case, depth_std


@pytest.mark.parametrize("engine", ENGINES)
@pytest.mark.parametrize("name", list(CASES))
def test_fused_render_edge_shape(name, engine):
    import pnr_native as pn
    case, depth_std = _case(name)
    cfg = case["cfg"]
    res = gpu_util.render_case_cuda(case, engine=engine, depth_std=depth_std)
    if engine != "simt":
        assert pn.tc_status() == 0
    fast = engine == "tc_fast"
    arith = fo.arithmetic if fast else None
    tols = dict(rgb_tol=fo.TIGHT_RGB, depth_tol=None, weights_tol=None) if fast else \
        dict(rgb_tol=1e-4, depth_tol=1e-4 if engine == "simt" else 2e-4, weights_tol=1e-4)
    # coarse pass: the stratified samples are exact, the outputs match the oracle at them
    r8 = case["rays"].reshape(-1, 8)
    zc_ref = gu.oracle.sample_coarse(r8, case["noise"]["u_coarse"], cfg["n_coarse"])
    assert (res["coarse"]["z"].cpu() - zc_ref).abs().max() < 1e-6
    coarse_errs = fpc.check_fine_outputs(case["rays"], res["coarse"]["z"], res["coarse"],
                                         fpc.case_composite(case, fine=False, arithmetic=arith), what="coarse",
                                         **dict(tols, depth_tol=None if fast else 1e-4))
    if cfg["n_fine"] == 0:
        assert "fine" not in res
        print(f"{name} {engine}: coarse {coarse_errs}")
        return
    chk = fpc.check_case(case, res, depth_std=depth_std, arithmetic=arith, **tols)
    print(f"{name} {engine}: {chk}  coarse {coarse_errs}")
    if name == "depth_clamps":
        z = res["fine"]["z"].cpu()
        assert (z == r8[:, 6:7]).any() and (z == r8[:, 7:8]).any(), "no depth sample clamped to near and to far"
