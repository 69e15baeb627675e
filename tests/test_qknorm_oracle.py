"""CPU checks of the q/k-norm + RoPE restatement (tests/qknorm_restatement.py) the GPU kernel is held to.

* HF's own Qwen3RMSNorm followed by apply_rotary_pos_emb (transformers' modeling_qwen3), on CPU in bf16 and fp16, equals
  one of the restatement's candidates on every element, and the nearest one wherever no rounding alternative exists;
* planted errors leave unexplained elements: the norm after RoPE, the q weight used for k, eps dropped, n not rounded
  before the weight, the mean over all heads of a row, the mean over half a head.
"""
import pytest
import torch

import qknorm_restatement as Q
from oracle import llama_ref as LR

DTYPES = {"bf16": torch.bfloat16, "fp16": torch.float16}
EPS = 1e-6


def _hf(x_q, x_k, wq, wk, eps, cos, sin):
    """HF's Qwen3 path on [R, H, D] heads: q_norm / k_norm, then apply_rotary_pos_emb on [1, H, R, D]."""
    from transformers.models.qwen3.modeling_qwen3 import Qwen3RMSNorm, apply_rotary_pos_emb
    D = x_q.shape[-1]
    qn, kn = Qwen3RMSNorm(D, eps=eps), Qwen3RMSNorm(D, eps=eps)
    with torch.no_grad():
        qn.weight.data = wq.clone()
        kn.weight.data = wk.clone()
        q = qn(x_q).transpose(0, 1)[None]
        k = kn(x_k).transpose(0, 1)[None]
        q, k = apply_rotary_pos_emb(q, k, cos[None], sin[None])
    return q[0], k[0]                                        # [H, R, D]


def _case(dtype, D, seed, rows=48, nh=8, nkv=4):
    g = torch.Generator().manual_seed(seed)
    xq, xk = Q.data(rows, nh, D, dtype, g), Q.data(rows, nkv, D, dtype, g)
    wq, wk = Q.weights(D, dtype, g), Q.weights(D, dtype, g)
    cos_t, sin_t = LR.rope_tables(D, 4096, 1e6, dtype, "cpu")
    pos = torch.randint(0, 4096, (rows,), generator=g)
    return xq, xk, wq, wk, cos_t[pos], sin_t[pos]


def _restated(x, w, eps, cos, sin, dtype):
    return Q.candidates(x.transpose(0, 1), w, eps, cos, sin, dtype)     # [4, H, R, D]


@pytest.mark.parametrize("D", [128, 64])
@pytest.mark.parametrize("dtn", list(DTYPES))
def test_restatement_equals_hf_qwen3_norm_and_rope(dtn, D):
    dtype = DTYPES[dtn]
    took = 0
    for seed in range(3):
        xq, xk, wq, wk, cos, sin = _case(dtype, D, seed)
        hq, hk = _hf(xq, xk, wq, wk, EPS, cos, sin)
        for got, x, w in ((hq, xq, wq), (hk, xk, wk)):
            cands = _restated(x, w, EPS, cos, sin, dtype)
            assert Q.unexplained(got, cands) == 0
            ambiguous = (cands != cands[0]).any(0)
            assert torch.equal(got[~ambiguous], cands[0][~ambiguous]), "HF differs where no rounding alternative exists"
            took += int((got != cands[0]).sum())
    print(f"{dtn} D {D}: {took} elements of HF's output took a rounding alternative")


def _planted(plant, x, w, w_other, eps, cos, sin, dtype):
    """[R, H, D] inputs, the restatement with one error planted; [H, R, D] output."""
    xd = x.double()
    D = x.shape[-1]
    eps32 = float(torch.tensor(eps, dtype=torch.float32))
    if plant == "norm_after_rope":
        r = Q.rope(x.transpose(0, 1), cos, sin).transpose(0, 1)
        main, _ = Q.norm_candidates(r, w, eps, dtype)
        return main.transpose(0, 1)
    if plant == "q_weight_for_k":
        return Q.candidates(x.transpose(0, 1), w_other, eps, cos, sin, dtype)[0]
    if plant == "eps_dropped":
        return Q.candidates(x.transpose(0, 1), w, 0.0, cos, sin, dtype)[0]
    if plant == "mean_over_row":
        ms = xd.pow(2).mean(dim=(-2, -1), keepdim=True)
    elif plant == "mean_over_half_head":
        ms = xd[..., : D // 2].pow(2).mean(-1, keepdim=True)
    else:
        ms = xd.pow(2).mean(-1, keepdim=True)
    v = xd / torch.sqrt(ms + eps32)
    n = v if plant == "n_unrounded" else v.to(dtype).double()
    y = (w.double() * n).to(dtype)
    return Q.rope(y.transpose(0, 1), cos, sin)


@pytest.mark.parametrize("plant", ["norm_after_rope", "q_weight_for_k", "eps_dropped", "n_unrounded", "mean_over_row",
                                   "mean_over_half_head"])
@pytest.mark.parametrize("dtn", list(DTYPES))
def test_planted_errors_leave_unexplained_elements(plant, dtn):
    dtype = DTYPES[dtn]
    xq, xk, wq, wk, cos, sin = _case(dtype, 128, 7)
    _, hk = _hf(xq, xk, wq, wk, EPS, cos, sin)
    cands = _restated(xk, wk, EPS, cos, sin, dtype)
    assert Q.unexplained(hk, cands) == 0
    bad = _planted(plant, xk, wk, wq, EPS, cos, sin, dtype)
    n_bad = Q.unexplained(bad, cands)
    print(f"{dtn} {plant}: {n_bad} of {bad.numel()} elements unexplained")
    assert n_bad > 0
