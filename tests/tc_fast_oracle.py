"""CPU restatement of the single-pass tensor engine (PNR_ENGINE_TC_FAST, engine "tc_fast") -- test infrastructure.

The single-pass kernel evaluates lin_in, fc_0 and fc_1 of every ResNet block as ONE fp16 tensor product per GEMM:
D += Ahi * Whi with fp32 accumulation, where Whi = fp16(W * s) of the packed image (s = the pack's power-of-two weight
scale, csrc/pnr_field_tc.cu k_pack_header) and Ahi = fp16(A) of the operand (saturating to +-65504).  Everything else
is the exact engine's arithmetic: lin_z through the fp32 projected-latent maps, the view mean, lin_out in fp32, the
output activations, compositing and resampling.  `resnetfc_fast` restates that; products of fp16 values are exact, so
they are summed in float64 and rounded once to fp32.  With products=3 it adds back the two correction products the
exact engine issues (Alo * Whi + Ahi * Wlo), i.e. it restates PNR_ENGINE_TC.

The bounds below are the ones tests/test_gpu_tc_fast.py enforces and tests/test_tc_fast_oracle.py checks this
restatement against; DESIGN.md 3.1 gives the measured values they were set from.
"""
import contextlib
import math

import torch
import torch.nn.functional as F

import golden_util as gu

oracle = gu.oracle

# Single-pass engine (GPU or this restatement) vs the fp32 oracle, golden cases: max |d rgb| of the coarse pass and of
# the fine pass at the kernel's own samples (tests/fine_pass_check.py); field values |d| / (1 + |ref|).  Measured on an
# H100 (c2/c3/c4_small): rgb up to 6.7e-3, field up to 8.9e-3.
LOOSE_RGB = 1.5e-2
LOOSE_FIELD = 3e-2
# GPU single-pass kernel vs this restatement.  Rounding every activation to fp16 makes the single pass sensitive to the
# last bit of its fp32 sums: this restatement with fp32 instead of float64 sums moves c4_small's field by 1.6e-3, so
# the kernel (tensor-core accumulation order) cannot follow it more closely than a few 1e-3.  Measured on an H100:
# rgb up to 2.0e-3, field up to 8.8e-3.  A wrong weight tile, ring slot or operand half gives errors of order 1e-1.
TIGHT_RGB = 5e-3
TIGHT_FIELD = 2e-2


def weight_scale(w):
    """The pack's power-of-two scale: 2^clamp(floor(log2(16384 / max|W|)), 0, 12) over lin_in, fc_0 and fc_1."""
    m = max(float(v.abs().max()) for k, v in w.items()
            if k.endswith("weight") and (k.startswith("lin_in") or ".fc_" in k))
    if not (m > 0 and math.isfinite(m)):
        return 1.0
    return 2.0 ** max(0, min(12, math.floor(math.log2(16384.0 / m))))


def _f16(x):
    return x.clamp(-65504.0, 65504.0).half().double()


def _linear(a, wt, b, scale, products):
    """y = (A W^T) + b on fp16 operands, as one tensor pass (products=1) or the three-pass split (products=3)."""
    ws = wt.double() * scale
    a_hi, w_hi = _f16(a), _f16(ws)
    acc = a_hi @ w_hi.t()
    if products == 3:
        a_lo, w_lo = _f16(a.double() - a_hi), _f16(ws - w_hi)
        acc = acc + a_lo @ w_hi.t() + a_hi @ w_lo.t()
    return (acc.float() / scale) + b


def resnetfc_fast(w, zx, NS, P, products=1, d_latent=512, n_blocks=5, combine_layer=3):
    """oracle.resnetfc with lin_in, fc_0 and fc_1 on the tensor engine's fp16 operands (lin_z and lin_out exact)."""
    scale = weight_scale(w)
    z = zx[..., :d_latent]
    x = _linear(zx[..., d_latent:], w["lin_in.weight"], w["lin_in.bias"], scale, products)
    for blk in range(n_blocks):
        if blk == combine_layer and NS > 1:
            x = x.reshape(-1, NS, P, x.shape[-1]).mean(dim=1).reshape(-1, x.shape[-1])
        if blk < combine_layer:
            x = x + F.linear(z, w[f"lin_z.{blk}.weight"], w[f"lin_z.{blk}.bias"])
        net = _linear(torch.relu(x), w[f"blocks.{blk}.fc_0.weight"], w[f"blocks.{blk}.fc_0.bias"], scale, products)
        x = x + _linear(torch.relu(net), w[f"blocks.{blk}.fc_1.weight"], w[f"blocks.{blk}.fc_1.bias"], scale,
                        products)
    return F.linear(torch.relu(x), w["lin_out.weight"], w["lin_out.bias"])


@contextlib.contextmanager
def arithmetic(products=1):
    """Runs the oracle's field evaluation on resnetfc_fast (oracle.field_eval looks resnetfc up at call time)."""
    orig = oracle.resnetfc
    oracle.resnetfc = lambda w, zx, NS, P, **kw: resnetfc_fast(w, zx, NS, P, products)
    try:
        yield
    finally:
        oracle.resnetfc = orig


def render(case, products=1):
    """gu.oracle_render(case) on the single-pass arithmetic."""
    with arithmetic(products), torch.no_grad():
        return gu.oracle_render(case)


def field_eval(xyz, viewdirs, state, latent, w, NS, products=1):
    """oracle.field_eval on the single-pass arithmetic."""
    with arithmetic(products), torch.no_grad():
        return oracle.field_eval(xyz, viewdirs, state, latent, w, NS)


def field(case, xyz, dirs, coarse=True, products=1):
    """PixelNeRFNet.forward of a golden case at xyz, dirs (SB,P,3) on the single-pass arithmetic -> (SB,P,4)."""
    w = case["wc"] if (coarse or case["wf"] is None) else case["wf"]
    return field_eval(xyz, dirs, gu.oracle_state(case), case["latent"], w, case["cfg"]["NS"], products)


def flipped_rays(z_a, z_b, tol=2e-4):
    """Fine-pass rays whose merged samples differ: an importance sample moved to another CDF bin."""
    return ((z_a - z_b).abs() > tol).any(dim=-1)


def render_errors(res, ref):
    """max |d rgb| of the coarse pass, of the fine pass on rays that kept their bins, and the flipped-ray count."""
    out = {"coarse": float((res["coarse"]["rgb"] - ref["coarse"]["rgb"]).abs().max())}
    if "fine" in ref:
        fl = flipped_rays(res["fine"]["z"], ref["fine"]["z"])
        d = (res["fine"]["rgb"] - ref["fine"]["rgb"])[~fl]
        out["fine"] = float(d.abs().max()) if d.numel() else 0.0
        out["flipped"] = int(fl.sum())
        out["rays"] = int(fl.numel())
    return out
