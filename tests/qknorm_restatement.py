"""Host restatement of lade_rope_append_qknorm (include/lade_sm100.h): Qwen3's per-head q/k RMSNorm, then the rotary
embedding, with the kernel's rounding points.

* ``norm_candidates``: y = T(w * T(x * rstd)) per head of D elements, through ``oracle.llama_ref.rms_norm_fp64`` (float64
  with the rounding alternative of n where x * rstd lies near a rounding midpoint).
* ``rope``: (y * cos) + (rotate_half(y) * sin) with every op in the model dtype, as tests/test_gpu_layer_ops.py states it.
* ``candidates``: the RoPE output of every combination of the two inputs an output element reads (y[j] and y[j +- D/2],
  each the nearest rounding or its alternative): [4, ...].  A correct output equals one of them.
* ``data``: heads drawn with their own scale, from 1e-3 (where eps matters) to 10, and norm weights in [0.5, 2].
"""
import torch

from oracle import llama_ref as LR


def norm_candidates(x: torch.Tensor, w: torch.Tensor, eps: float, dtype):
    """(main, alt) of the per-head norm of x [..., D] with weight w [D], both in `dtype`."""
    D = x.shape[-1]
    _, main, alt = LR.rms_norm_fp64(x.reshape(-1, D), None, w, eps, dtype)
    return main.view(x.shape), alt.view(x.shape)


def rope(y: torch.Tensor, cos: torch.Tensor, sin: torch.Tensor) -> torch.Tensor:
    """y [..., R, D] in the model dtype, cos / sin [R, D]: every product and the sum rounded to the model dtype."""
    return (y * cos) + (LR.rotate_half(y) * sin)


def candidates(x: torch.Tensor, w: torch.Tensor, eps: float, cos, sin, dtype) -> torch.Tensor:
    """[4, ...]: RoPE of (main or alt at the element itself) x (main or alt at its partner across the half)."""
    main, alt = norm_candidates(x, w, eps, dtype)
    half = x.shape[-1] // 2
    out = []
    for own in (main, alt):
        for partner in (main, alt):
            # element j reads y[j] (own) and y[j -+ half] (partner): take `own` at j, `partner` at the other half
            lo = torch.cat([own[..., :half], partner[..., half:]], dim=-1)
            hi = torch.cat([partner[..., :half], own[..., half:]], dim=-1)
            r_lo, r_hi = rope(lo, cos, sin), rope(hi, cos, sin)
            out.append(torch.cat([r_lo[..., :half], r_hi[..., half:]], dim=-1))
    return torch.stack(out)


def unexplained(got: torch.Tensor, cands: torch.Tensor) -> int:
    """Elements of `got` that equal none of the candidates (NaN equals NaN)."""
    hit = torch.zeros_like(got, dtype=torch.bool)
    for c in cands:
        hit |= (got == c) | (torch.isnan(got) & torch.isnan(c))
    return int((~hit).sum())


def data(rows: int, heads: int, D: int, dtype, gen, device="cpu") -> torch.Tensor:
    """[rows, heads, D]: randn per head times a log-uniform scale in [1e-3, 10]."""
    x = torch.randn(rows, heads, D, generator=gen, device=device)
    scale = torch.exp(torch.empty(rows, heads, 1, device=device).uniform_(-6.9, 2.3, generator=gen))
    return (x * scale).to(dtype)


def weights(D: int, dtype, gen, device="cpu") -> torch.Tensor:
    return torch.empty(D, device=device).uniform_(0.5, 2.0, generator=gen).to(dtype)
