"""The mesh-extraction oracle against the unmodified reference (tests/golden/recon_ns*.npz, oracle/make_golden_recon.py):
the evaluation grid of util.gen_grid bit for bit, the fake view directions of recon.py:54, and the field the reference's
network gives on them."""
import numpy as np
import pytest
import torch

import golden_util as gu
from recon_util import recon

GRIDS = ("box", "odd", "flat")


def load(ns):
    return np.load(f"{gu.GOLD}/recon_ns{ns}.npz")


def ulp_diff(a, b):
    ia = a.view(np.int32).astype(np.int64)
    ib = b.view(np.int32).astype(np.int64)
    ia = np.where(ia < 0, np.int64(-2 ** 31) - ia, ia)
    ib = np.where(ib < 0, np.int64(-2 ** 31) - ib, ib)
    return np.abs(ia - ib)


@pytest.mark.parametrize("ns", [1, 2])
@pytest.mark.parametrize("grid", GRIDS)
def test_grid_points_and_directions(ns, grid):
    z = load(ns)
    pts = recon.grid_points(z[grid + "/lo"], z[grid + "/hi"], z[grid + "/reso"])
    assert pts.dtype == np.float32
    assert np.array_equal(pts.view(np.int32), z[grid + "/points"].view(np.int32))
    d, ref = recon.fake_viewdirs(pts), z[grid + "/dirs"]
    nan = np.isnan(ref)
    assert np.array_equal(np.isnan(d), nan)
    assert ulp_diff(d[~nan], ref[~nan]).max() <= 2
    if grid == "odd":
        assert nan.any(axis=1).sum() == 1 and not pts[nan.any(axis=1)].any()     # the origin, and only there


@pytest.mark.parametrize("ns", [1, 2])
@pytest.mark.parametrize("grid", GRIDS)
def test_oracle_field_matches_reference_sigma(ns, grid):
    z = load(ns)
    case = gu.load_case(str(z["case"]))
    src = case["src_poses"][:, :ns]
    state = gu.oracle.encode_state(src.reshape(-1, 4, 4), case["focal"], case["c"], case["cfg"]["W"],
                                   case["cfg"]["H"])
    pts = torch.from_numpy(z[grid + "/points"])[None]
    dirs = torch.from_numpy(z[grid + "/dirs"])[None]
    for key, w in (("coarse", case["wc"]), ("fine", case["wf"])):
        out = gu.oracle.field_eval(pts, dirs, state, case["latent"][:ns], w, ns)[0].numpy()
        ref = z[f"{grid}/{key}"]
        fin = np.isfinite(ref[:, 3])
        assert fin.sum() >= len(ref) - 1
        assert ref[fin, 3].max() > 0                          # a visible field, not all-zero sigma
        # relative to the field's scale: fp32 sums in another order differ by a few ulp of the largest sigma
        err = np.abs(out[fin, 3] - ref[fin, 3]).max() / (1.0 + np.abs(ref[fin, 3]).max())
        assert err <= 1e-5, (key, err)
