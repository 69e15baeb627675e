"""Cost of the FP8 projection GEMM at the decode shapes (DESIGN.md §7.2).

Each projection alone (m = 120 and 240; 7B and 13B (N, K)): lade_gemm_fp8, cuBLAS bf16 (torch.mm), torch._scaled_mm
with row-wise scales, and the library's lade_gemm_bf16 (m <= 128 only), as the median of CUDA-event timed rounds of 20
launches, the four alternating inside each round; and the achieved weight-streaming bandwidth.  A library call that
returns an error stops the script instead of being timed.

Prints the card and its power limit first.  Usage: python tools/fp8_gemm_cost.py [--rounds 7]
"""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests"))

SHAPES = {"7B": dict(hidden=4096, inter=11008), "13B": dict(hidden=5120, inter=13824)}


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip()


def timed(fn, reps=20):
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    fn()
    s.record()
    for _ in range(reps):
        fn()
    e.record()
    e.synchronize()
    return s.elapsed_time(e) / reps * 1e3     # us


def gemm_costs(rounds):
    import fp8_restatement as F
    from lookaheaddecoding_b200 import _cabi
    lib = _cabi.load()
    st = torch.cuda.current_stream().cuda_stream
    out = []
    for name, c in SHAPES.items():
        H, I = c["hidden"], c["inter"]
        for pn, (n, k) in dict(qkv=(3 * H, H), o=(H, H), gate_up=(2 * I, H), down=(H, I)).items():
            w = (torch.randn(n, k, device="cuda") * 0.02).to(torch.bfloat16)
            qw, sw = F.quant_rows(w.float())
            wt = qw.view(torch.float8_e4m3fn)
            for m in (120, 240):
                a = torch.randn(m, k, device="cuda").to(torch.bfloat16)
                qa, sa = F.quant_rows(a.float())
                cb = torch.empty(m, n, dtype=torch.bfloat16, device="cuda")
                fns = {
                    "gemm_fp8": lambda: _cabi.check(lib.lade_gemm_fp8(st, qa.data_ptr(), sa.data_ptr(), qw.data_ptr(),
                                                                      sw.data_ptr(), cb.data_ptr(), m, m, n, k, n, 0, 0),
                                                    "lade_gemm_fp8"),
                    "cublas_bf16": lambda: torch.mm(a, w.t(), out=cb),
                    "scaled_mm": lambda: torch._scaled_mm(qa.view(torch.float8_e4m3fn), wt.t(), scale_a=sa[:, None],
                                                          scale_b=sw[None, :], out_dtype=torch.bfloat16),
                }
                if m <= 128:
                    fns["gemm_bf16"] = lambda: _cabi.check(lib.lade_gemm_bf16(st, a.data_ptr(), w.data_ptr(), cb.data_ptr(),
                                                                              m, m, n, k, n, 0, 0), "lade_gemm_bf16")
                res = {kk: [] for kk in fns}
                for _ in range(rounds):
                    for kk, fn in fns.items():
                        try:
                            res[kk].append(timed(fn))
                        except RuntimeError as ex:     # a torch build without row-wise _scaled_mm; LadeError re-raises
                            if isinstance(ex, _cabi.LadeError):
                                raise
                            res[kk].append(float("nan"))
                            print(f"{kk}: {ex}", file=sys.stderr)
                med = {kk: sorted(v)[len(v) // 2] for kk, v in res.items()}
                bw = {"gemm_fp8": n * k / (med["gemm_fp8"] * 1e-6) / 1e12,
                      "cublas_bf16": 2 * n * k / (med["cublas_bf16"] * 1e-6) / 1e12}
                row = dict(model=name, proj=pn, m=m, N=n, K=k, us={kk: round(v, 1) for kk, v in med.items()},
                           TBps={kk: round(v, 2) for kk, v in bw.items()})
                print(json.dumps(row), flush=True)
                out.append(row)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=7)
    a = ap.parse_args()
    print(json.dumps({"card": card()}), flush=True)
    gemm_costs(a.rounds)


if __name__ == "__main__":
    main()
