#!/usr/bin/env python
"""Per-CTA phase timeline of the wgmma attention kernel (lade_debug_attn_timing).

The kernel stamps %globaltimer (ns, one clock for the whole GPU, so CTAs on different SMs compare) at fixed phases and
records the SM it ran on in slot 15.  Reported per shape: the start spread of the CTAs, whether any CTA started on an
SM only after another CTA of the same launch had finished there (a second round), and the median time from a CTA's
start to each of its phases.  `timer_step_ns` is the smallest non-zero difference between any two stamps: differences
below it are not resolved."""
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from lookaheaddecoding_b200 import _cabi  # noqa: E402
from attn_microbench import steady_rowmask  # noqa: E402

PHASES = ["start", "kfull0", "sfull0", "ofinal", "staged", "ticket", "merged", "end"]


def main():
    lib = _cabi.load()
    H, D, L = 32, 128, 8
    for kv, ns in [(1024, 4), (1278, 4), (3072, 4)]:
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
            _cabi.check(lib.lade_attn_fwd(st, q.data_ptr(), kvc[l, 0].data_ptr(), kvc[l, 1].data_ptr(), out.data_ptr(),
                                          rd.data_ptr(), mw, meta.data_ptr(), scratch.data_ptr(), q_len, H, H, D, cap,
                                          kv + q_len, ns, 2))
        for l in range(L):
            run(l)
        torch.cuda.synchronize()
        _cabi.check(lib.lade_debug_attn_timing(tb.data_ptr()))
        run(0)
        torch.cuda.synchronize()
        _cabi.check(lib.lade_debug_attn_timing(0))
        t = tb.cpu().numpy().reshape(-1, 16)                       # CTA order: head-major, split fastest
        t = t[t[:, 0] > 0]
        sm = t[:, 15]
        stamps = t[:, :8].astype(np.float64)
        start, end = stamps[:, 0], stamps[:, 7]
        vals = np.unique(t[:, :8][t[:, :8] > 0])
        step = int(np.diff(vals).min()) if len(vals) > 1 else 0
        # a second round: some CTA starts on an SM after another CTA of this launch has ended there
        second = 0
        for s in np.unique(sm):
            idx = np.where(sm == s)[0]
            for i in idx:
                if any(start[i] >= end[j] for j in idx if j != i):
                    second += 1
        rel = {}
        for i, n in enumerate(PHASES):
            ok = stamps[:, i] > 0
            if ok.any():
                rel[n] = round(float(np.median(stamps[ok, i] - start[ok])) / 1e3, 2)
        print(json.dumps({"kv": kv, "splits": ns, "ctas": int(len(t)), "sms_used": int(len(np.unique(sm))),
                          "timer_step_ns": step, "start_spread_us": round(float(start.max() - start.min()) / 1e3, 2),
                          "launch_span_us": round(float(end.max() - start.min()) / 1e3, 2),
                          "ctas_in_second_round": second,
                          "last_start_us": round(float(np.sort(start)[-1] - start.min()) / 1e3, 2),
                          "median_us_since_cta_start": rel}))


if __name__ == "__main__":
    main()
