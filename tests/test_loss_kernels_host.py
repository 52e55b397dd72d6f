"""The loss-kernel bounds of loss_ref.py are tight enough to catch real faults (runs on the CPU).

For each deliberate fault the test computes the float64 reference of the faulty kernel on inputs of
test_loss_kernels_gpu.py and checks that it misses the unmutated bound by at least 10x on some element.  It also pins
the reference's loss to the fp32 oracle's formulas run in float64."""
import math

import pytest
import torch
from loss_ref import (EPS_F32, F64, egonce_reference, f32, fused_case, maxmargin_case, maxmargin_reference, nce_case,
                      nce_reference, normalise)

from oracle import reference_port as rp

MIN_FACTOR = 10.0


def factor(name, got, ref, bound):
    f = ((got.to(F64) - ref).abs() / bound.clamp_min(1e-300)).nan_to_num(nan=math.inf).max().item()
    print(f"[mutant] {name}: exceeds the bound by {f:.3g}x")
    return f


@pytest.mark.parametrize("mode", [0, 1, 2, 3])
def test_reference_loss_matches_oracle_formulas(mode):
    t, v, verb, noun, mask, temp = fused_case(40, 33, mode, 118, 582, 3, "train")
    r = egonce_reference(t, v, mask, f32(1 / temp), "fused")
    x = rp.sim_matrix(t.double(), v.double(), EPS_F32)
    sv, sn = rp.sim_matrix(verb.double(), verb.double()), rp.sim_matrix(noun.double(), noun.double())
    if mode == 0:
        want = rp.norm_softmax_loss(x, 1 / f32(1 / temp))
    else:
        want = rp.egonce_loss(x, sv, sn, 1 / f32(1 / temp), noun=mode in (1, 2), verb=mode in (1, 3))
    assert abs(r["loss"].item() - want.item()) <= 1e-12 * max(1.0, abs(want.item()))


@pytest.mark.parametrize("fix_norm", [True, False])
def test_maxmargin_reference_matches_oracle(fix_norm):
    x, w = maxmargin_case(33, 5, adaptive=True)
    for weight in (None, w):
        r = maxmargin_reference(x, 0.25, fix_norm, weight)
        xx = x.double().requires_grad_(True)
        want = (rp.max_margin_ranking_loss(xx, 0.25, fix_norm) if weight is None
                else rp.adaptive_max_margin_ranking_loss(xx, weight.double(), 0.25, fix_norm))
        want.backward()
        assert abs(r["loss"].item() - want.item()) <= 1e-14
        assert torch.allclose(r["dx"], xx.grad, rtol=1e-12, atol=1e-15)
        assert torch.equal(r["dx"] == 0, xx.grad == 0)


def test_mutants_exceed_bounds():
    found = {}
    # (a) the column LSE over the transposed mask (non-symmetric mask, nce_* path)
    x, mask, temp = nce_case(33, 11)
    it = f32(1 / temp)
    ref = nce_reference(x, mask, it)
    mut = nce_reference(x, mask, it, col_mask=mask.T)
    found["a: column LSE over mask^T"] = factor("a", mut["stats"], ref["stats"], ref["stats_err"])

    # (b) the diagonal not forced positive (fused path, training regime, mode 1)
    t, v, verb, noun, mask, temp = fused_case(65, 256, 1, 118, 582, 2, "train")
    it = f32(1 / temp)
    ref = egonce_reference(t, v, mask, it, "fused")
    eye = torch.eye(65, dtype=torch.bool)
    mut = egonce_reference(t, v, mask & ~eye, it, "fused")
    found["b: diagonal not positive"] = factor("b", mut["stats"], ref["stats"], ref["stats_err"])

    # (c) |a| + eps instead of max(|a|, eps): seen on the near-zero rows
    def plus_eps(a, eps):
        a = a.to(F64)
        n = a.norm(dim=1)
        return a / (n + eps)[:, None], n
    mut = egonce_reference(t, v, mask, it, "fused", norm_fn=plus_eps)
    found["c: norm + eps"] = max(factor("c stats", mut["stats"], ref["stats"], ref["stats_err"]),
                                 factor("c d_text", mut["d_text"], ref["d_text"], ref["d_text_err"]))

    # (d) the last row and column of a partial 32-tile dropped (G = 33): the other rows' and columns' statistics
    t, v, verb, noun, mask, temp = fused_case(33, 32, 1, 118, 582, 4, "gauss")
    it = f32(1 / temp)
    ref = egonce_reference(t, v, mask, it, "fused")
    mut = egonce_reference(t[:32], v[:32], mask[:32, :32], it, "fused")
    keep = torch.cat([torch.arange(32) + k * 33 for k in range(4)])
    found["d: last row / column dropped"] = factor("d", mut["stats"], ref["stats"][keep], ref["stats_err"][keep])

    # (e) the backward without the column-softmax term; (f) the row-normalisation backward without the projection
    t, v, verb, noun, mask, temp = fused_case(64, 256, 1, 118, 582, 6, "train")
    it = f32(1 / temp)
    ref = egonce_reference(t, v, mask, it, "fused")
    la_r, lp_r = ref["stats"][:64], ref["stats"][64:128]
    z = ref["z"]
    dx_rows = -(it / 64) * (mask.double() * torch.exp(z - lp_r[:, None]) - torch.exp(z - la_r[:, None]))
    _, nt = normalise(t)
    tn = ref["tn"]
    d_text = torch.where((nt > EPS_F32)[:, None], (dx_rows @ ref["vn"] - tn * ((dx_rows @ ref["vn"]) * tn).sum(1,
                         keepdim=True)) / nt.clamp_min(EPS_F32)[:, None], dx_rows @ ref["vn"] / EPS_F32)
    found["e: no column-softmax term"] = factor("e", d_text, ref["d_text"], ref["d_text_err"])
    dan = ref["dx"] @ ref["vn"]
    d_text = torch.where((nt > EPS_F32)[:, None], dan / nt.clamp_min(EPS_F32)[:, None], dan / EPS_F32)
    found["f: no projection"] = factor("f", d_text, ref["d_text"], ref["d_text_err"])

    # (g) max-margin counting i == j under fix_norm
    x, w = maxmargin_case(33, 7, adaptive=False)
    ref = maxmargin_reference(x, 0.25, True)
    mut_loss = ref["loss"] + 2 * 33 * f32(0.25) / (2 * 33 * 32)
    found["g: i == j counted"] = factor("g", mut_loss, ref["loss"], ref["loss_err"])

    weak = {k: f for k, f in found.items() if not f >= MIN_FACTOR}
    assert not weak, f"faults within {MIN_FACTOR}x of the bound: {weak}"
