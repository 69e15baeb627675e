#!/usr/bin/env python
"""Per-CTA phase timeline of the wgmma attention kernel (lade_debug_attn_timing)."""
import os, sys, json
import numpy as np
import torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from lookaheaddecoding_b200 import _cabi
from attn_microbench import steady_rowmask

lib = _cabi.load()
H, D, L = 32, 128, 8
for kv, ns in [(1024, 4), (3072, 4)]:
    rm_np, mw, q_len = steady_rowmask(15, 5, 15)
    cap = kv + q_len + 64
    kvc = torch.randn(L, 2, H, cap, D, device="cuda", dtype=torch.bfloat16)
    q = torch.randn(H, q_len, D, device="cuda", dtype=torch.bfloat16)
    out = torch.empty(q_len, H * D, device="cuda", dtype=torch.bfloat16)
    rd = torch.from_numpy(rm_np).cuda()
    meta = torch.zeros(_cabi.META_INTS, dtype=torch.int32, device="cuda")
    for k, v in {_cabi.M_Q_LEN: q_len, _cabi.M_KV_LEN: kv, _cabi.M_N_INPUT: 1, _cabi.M_PHASE: 2, _cabi.M_Q_PAD: q_len}.items():
        meta[k] = v
    scratch = torch.zeros(lib.lade_attn_scratch_bytes(q_len, H, D, ns), dtype=torch.uint8, device="cuda")
    tb = torch.zeros(ns * H * 16, dtype=torch.int64, device="cuda")
    st = torch.cuda.current_stream().cuda_stream
    def run(l):
        _cabi.check(lib.lade_attn_fwd(st, q.data_ptr(), kvc[l, 0].data_ptr(), kvc[l, 1].data_ptr(), out.data_ptr(), rd.data_ptr(), mw,
                                      meta.data_ptr(), scratch.data_ptr(), q_len, H, H, D, cap, kv + q_len, ns, 2))
    for l in range(L): run(l)
    torch.cuda.synchronize()
    _cabi.check(lib.lade_debug_attn_timing(tb.data_ptr()))
    run(0)
    torch.cuda.synchronize()
    _cabi.check(lib.lade_debug_attn_timing(0))
    t_all = tb.cpu().numpy().reshape(-1, 16).astype(np.float64)          # CTA order: head-major, split fastest
    per_split = {}
    for sp in range(ns):
        ts = t_all[sp::ns]
        ts = ts[ts[:, 0] > 0]
        if len(ts):
            per_split[sp] = {"ofinal": round(float(np.median((ts[:, 3] - ts[:, 0]) / 1.965e3)), 2),
                             "compute_done": round(float(np.median((ts[:, 4] - ts[:, 0]) / 1.965e3)), 2),
                             "start_skew": round(float(np.median((ts[:, 0] - t_all[0::ns][:len(ts), 0]) / 1.965e3)), 2)}
    t = t_all[t_all[:, 0] > 0]
    names = ["start", "kfull0", "sfull0", "ofinal", "compute_done", "barrier1", "pushed_barrier2", "end", "t1_begin", "t1_sfull", "t1_ld", "t1_max", "t1_bar", "t1_exp", "t1_fence", "t1_arrive"]
    rel = (t - t[:, :1]) / 1.965e3     # us at 1965 MHz
    print(json.dumps({"kv": kv, "splits": ns, "ctas": int(len(t)),
                      "median_us_since_start": {n: round(float(np.median(rel[:, i])), 2) for i, n in enumerate(names)
                                                if np.median(t[:, i]) > 0},
                      "per_split_us": per_split}))
