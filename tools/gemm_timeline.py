#!/usr/bin/env python
"""Per-CTA phase timeline of the wgmma projection GEMM (lade_debug_gemm_timing, %globaltimer ns).

Four back-to-back launches on distinct weights are replayed from a CUDA graph; for each launch the phases are
reported relative to the earliest CTA start of that launch, plus the idle gap to the previous launch's last exit.
"""
import argparse
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from lookaheaddecoding_b200 import _cabi  # noqa: E402
from gemm_microbench import SHAPES_7B  # noqa: E402

NAMES = ["start", "setup_done", "first_w_tile", "last_mma_issued", "acc_full", "epilogue_done", "cluster_sync", "end"]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--m", type=int, default=120)
    ap.add_argument("--shapes", nargs="+", default=["qkv", "o", "gate_up", "down"])
    ap.add_argument("--cfg", default="0:0")
    a = ap.parse_args()
    lib = _cabi.load()
    parts = [int(v) for v in a.cfg.split(":")]
    tn = parts[0] | ((parts[2] if len(parts) > 2 else 0) << 16) | ((parts[3] if len(parts) > 3 else 0) << 20)
    sk = parts[1]
    for name in a.shapes:
        n, k = SHAPES_7B[name]
        ws = [(torch.randn(n, k, device="cuda") * 0.02).to(torch.bfloat16) for _ in range(4)]
        x = torch.randn(128, k, device="cuda").to(torch.bfloat16)
        c = torch.empty(128, n, dtype=torch.bfloat16, device="cuda")
        tb = torch.zeros(4 * 1024 * 8, dtype=torch.int64, device="cuda")
        s = torch.cuda.Stream()
        with torch.cuda.stream(s):
            def run():
                for w in ws:
                    _cabi.check(lib.lade_gemm_bf16(s.cuda_stream, x.data_ptr(), w.data_ptr(), c.data_ptr(), a.m, 128, n, k, n, tn, sk))
            run()
            s.synchronize()
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g, stream=s):
                run()
        torch.cuda.synchronize()
        for _ in range(3):
            g.replay()
        torch.cuda.synchronize()
        _cabi.check(lib.lade_debug_gemm_timing(tb.data_ptr()))
        g.replay()
        torch.cuda.synchronize()
        _cabi.check(lib.lade_debug_gemm_timing(0))
        t = tb.cpu().numpy().reshape(4, 1024, 8).astype(np.float64)
        order = sorted(range(4), key=lambda i: t[i][t[i][:, 0] > 0][:, 0].min() if (t[i][:, 0] > 0).any() else 0)
        prev_end = None
        for i in order:
            ti = t[i][t[i][:, 0] > 0]
            if not len(ti):
                continue
            t0 = ti[:, 0].min()
            rel = (ti - t0) / 1e3
            rec = {"shape": name, "cfg": a.cfg, "ctas": int(len(ti)),
                   "gap_from_prev_end_us": None if prev_end is None else round((t0 - prev_end) / 1e3, 2),
                   "median_us": {nm: round(float(np.median(rel[:, j])), 2) for j, nm in enumerate(NAMES) if ti[:, j].max() > 0},
                   "max_us": {nm: round(float(rel[:, j].max()), 2) for j, nm in enumerate(NAMES) if ti[:, j].max() > 0}}
            prev_end = ti[:, 7].max()
            print(json.dumps(rec), flush=True)
        del ws


if __name__ == "__main__":
    main()
