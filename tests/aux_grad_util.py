"""Loads tests/golden/grad_aux_*.npz (oracle/make_golden_aux.py): the reference's gradients for a loss on
all six renderer outputs (rgb MSEs + its alpha loss on fine.weights.sum(-1) + depth MSEs + a coarse-weights term),
together with the upstream gradient of each output, so that a test can replay the backward without any loss code."""
import os

import numpy as np
import torch

import golden_util as gu

CASE_NAMES = ["tiny", "sb2_d"]
OUTPUTS = ("coarse.rgb", "coarse.depth", "coarse.weights", "fine.rgb", "fine.depth", "fine.weights")


def up_name(output):
    """'fine.weights' -> 'd_weights_fine' (the PnrRenderGrad / oracle render_backward key)."""
    p, q = output.split(".")
    return f"d_{q}_{p}"


def load(name):
    z = np.load(os.path.join(gu.GOLD, "grad_aux_" + name + ".npz"))
    t = lambda k: torch.from_numpy(z[k])
    return dict(loss=float(z["loss"]), rgb_gt=t("rgb_gt"), depth_gt=t("depth_gt"), g_latent=t("g_latent"),
                up={o: t("up/" + o) for o in OUTPUTS},
                gc={k[3:]: t(k) for k in z.files if k.startswith("gc/")},
                gf={k[3:]: t(k) for k in z.files if k.startswith("gf/")})


def flat_up(aux, R):
    """Upstream gradients keyed like PnrRenderGrad, flattened to [R][...] (depth: [R]) contiguous fp32."""
    out = {}
    for o, v in aux["up"].items():
        v = v.reshape(R, -1).float().contiguous()
        out[up_name(o)] = v.reshape(R).contiguous() if v.shape[1] == 1 else v
    return out


def rel(a, ref):
    return ((a - ref).abs().max() / (ref.abs().max() + 1e-20)).item()
