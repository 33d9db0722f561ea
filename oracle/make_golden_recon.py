"""
ORACLE TOOLING -- generates tests/golden/recon_ns{1,2}.npz by running the UNMODIFIED reference (imported through
oracle/ref_harness.py) on CPU: the evaluation grid and field of src/util/recon.py's marching_cubes.

    python oracle/make_golden_recon.py

Run where a reference checkout is readable (not on the GPU box).  The reference's own marching_cubes cannot run: it
needs PyMCubes, and it calls the network with 2-D points, which PixelNeRFNet.forward rejects.  So this records what it
would feed marching cubes, with the 3-D call it should have made:
  * points  util.gen_grid(*zip(c1, c2, reso), ij_indexing=True) (recon.py:43)
  * dirs    -grid / torch.norm(grid, dim=-1) (recon.py:54)
  * coarse / fine   net(points[None], coarse=..., viewdirs=dirs[None])[0], all four outputs
on the `tiny` case's weights, latent and cameras, with both source views (ns2) and with the first only (ns1).  The
grids are small and not cubic; `odd` has symmetric bounds whose linspace hits 0 exactly, so the origin is a grid point
(NaN view direction there).
"""
import importlib.util
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)


def _load(name, path):
    spec = importlib.util.spec_from_file_location(name, path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


mg = _load("pnr_make_golden", os.path.join(HERE, "make_golden.py"))
ref_harness = mg.ref_harness

GRIDS = {
    "box": ((-0.6, -0.5, -0.4), (0.7, 0.55, 0.45), (9, 7, 5)),
    "odd": ((-0.75, -0.75, -0.75), (0.75, 0.75, 0.75), (7, 5, 9)),
    "flat": ((-0.3, -0.45, -0.2), (0.35, 0.4, 0.25), (4, 11, 6)),
}
CASE = "tiny"


def recon_fixture(ns):
    cs = mg.CASES[CASE]
    inp = mg.case_inputs(CASE, cs)
    net, _ = ref_harness.build_reference(cs["d_hidden"], inp["wc"], inp["wf"], cs["n_coarse"], cs["n_fine"],
                                         cs["n_fine_depth"])
    _, _, util = ref_harness.import_reference()
    ref_harness.set_scene(net, inp["latent"][:ns], inp["src_poses"][:, :ns], inp["focal"], inp["c"], cs["W"], cs["H"])
    rec = dict(case=np.array(CASE), ns=np.array(ns))
    for name, (c1, c2, reso) in GRIDS.items():
        with torch.no_grad():
            grid = util.gen_grid(*zip(c1, c2, reso), ij_indexing=True)
            dirs = -grid / torch.norm(grid, dim=-1).unsqueeze(-1)
            coarse = net(grid[None], coarse=True, viewdirs=dirs[None])[0]
            fine = net(grid[None], coarse=False, viewdirs=dirs[None])[0]
        rec.update({f"{name}/lo": np.array(c1), f"{name}/hi": np.array(c2), f"{name}/reso": np.array(reso),
                    f"{name}/points": grid.numpy(), f"{name}/dirs": dirs.numpy(), f"{name}/coarse": coarse.numpy(),
                    f"{name}/fine": fine.numpy()})
    path = os.path.join(mg.GOLD, f"recon_ns{ns}.npz")
    np.savez_compressed(path, **rec)
    print(f"recon_ns{ns}: wrote {path} ({os.path.getsize(path) / 1e3:.0f} KB)")


if __name__ == "__main__":
    os.makedirs(mg.GOLD, exist_ok=True)
    for ns in (1, 2):
        recon_fixture(ns)
