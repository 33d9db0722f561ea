"""The CPU restatement of the single-pass tensor engine (tests/tc_fast_oracle.py), which tests/test_gpu_tc_fast.py
holds the GPU kernel to, checked against the fp32 oracle (no GPU needed)."""
import pytest
import torch

import golden_util as gu
import tc_fast_oracle as fo

CASES = ["c2_small", "c3_small", "c4_small"]   # the d_hidden = 512 golden cases (the tensor engine's shape)


def test_cases_are_tensor_engine_shapes():
    for name in CASES:
        assert gu.load_case(name)["cfg"]["d_hidden"] == 512, name
    assert gu.load_case("sb2_d")["cfg"]["d_hidden"] == 32     # the GPU test's refusal case: no tensor engine shape


def test_weight_scale_is_the_packs():
    w = {"lin_in.weight": torch.tensor([[0.5, -3.0]]), "blocks.0.fc_0.weight": torch.tensor([[1.0]]),
         "lin_z.0.weight": torch.tensor([[1e6]]), "lin_out.weight": torch.tensor([[1e6]])}
    assert fo.weight_scale(w) == 2.0 ** 12        # floor(log2(16384 / 3)) = 12, the cap; lin_z / lin_out not packed
    w["blocks.0.fc_0.weight"] = torch.tensor([[300.0]])
    assert fo.weight_scale(w) == 2.0 ** 5         # floor(log2(54.6)) = 5


def test_three_products_restate_the_exact_engine():
    """With the two dropped products added back the restatement is the exact engine's split arithmetic: it reproduces
    the fp32 oracle to split precision, so the single pass's error is the dropped products and nothing else."""
    case = gu.load_case("c2_small")
    ref = gu.oracle_render(case)
    err = fo.render_errors(fo.render(case, products=3), ref)
    assert err["coarse"] < 1e-5 and err["fine"] < 1e-5, err
    assert err["flipped"] == 0, err
    r = case["ref"]
    out = fo.field(case, r["field_xyz"], r["field_dirs"], coarse=True, products=3)
    assert ((out - r["field_coarse"]).abs() / (1 + r["field_coarse"].abs())).max() < 1e-4


@pytest.mark.parametrize("name", CASES)
def test_single_pass_error_within_the_gpu_bounds(name):
    """Render and field of the single pass against the fp32 oracle stay within the loose bounds the GPU test uses,
    and differ from it by clearly more than split precision (the restatement really drops the products)."""
    case = gu.load_case(name)
    ref = gu.oracle_render(case)
    err = fo.render_errors(fo.render(case), ref)
    print(name, err)
    assert 1e-5 < err["coarse"] < fo.LOOSE_RGB, err
    if "fine" in err:
        assert err["fine"] < fo.LOOSE_RGB, err
    r = case["ref"]
    for coarse, key in ((True, "field_coarse"), (False, "field_fine")):
        out = fo.field(case, r["field_xyz"], r["field_dirs"], coarse=coarse)
        rel = ((out - r[key]).abs() / (1 + r[key].abs())).max().item()
        assert rel < fo.LOOSE_FIELD, (key, rel)
