#!/usr/bin/env python
"""Where does the steady decode step go, IN the graph (warm caches, real launch gaps)?  ncu serialises and flushes,
so its per-kernel times overstate the small kernels.  Here the captured step graph is rebuilt with one kernel family
left out at a time (results are garbage, timing is not) and replayed back to back; the difference to the full step is
what that family costs in situ, launch gaps included.  A family is left out by replacing the engine's stage method with
a no-op; `gemm` is every projection, the lm_head GEMM included."""
import json
import os
import random
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import bench  # noqa: E402
from lookaheaddecoding_b200 import LookaheadEngine  # noqa: E402

STAGES = {"norm": "_norm", "gemm": "_proj", "rope": "_rope_append", "attn": "_attention", "swiglu": "_swiglu"}


@torch.no_grad()
def main():
    shape = bench.WORKLOADS["7b"][0]
    dev = torch.device("cuda", 0)
    model = bench.build_model(shape, dev)
    W, N, G, P, new = 15, 5, 15, 1024, 256
    eng = LookaheadEngine(model, W, N, G, max_total_len=P + new + 8)
    torch.manual_seed(1)
    prompt = torch.randint(3, shape["vocab"], (P,)).tolist()
    eng.generate(prompt, 130, rng=random.Random(0))       # kv ~ 1150 afterwards: mid-run context

    def ablate(families):
        for name in STAGES.values():                       # instance attributes shadow the class's stage methods
            eng.__dict__.pop(name, None)
        for f in families:
            setattr(eng, STAGES[f], lambda *args: 0)

    def graph_ms(families, reps=60):
        eng._graph = None
        eng.begin(prompt, P + new, (), eng.draw_window(prompt, random.Random(0), None))
        ablate(())
        for s in range(N - 2):                             # real prefill + window fill so that kv_len / phase are steady
            eng.run_forward_step(s, P)
            eng._read_result()
        ablate(families)
        g = eng._steady_graph(True)
        for _ in range(5):
            g.replay()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(reps):
            g.replay()
        e1.record()
        torch.cuda.synchronize()
        ablate(())
        return e0.elapsed_time(e1) / reps

    full = graph_ms(())
    out = {"full_step_ms": round(full, 4), "per_layer_us": round(full * 1e3 / eng.L, 2)}
    for name in ("rope", "attn", "norm", "swiglu", "gemm"):
        ms = graph_ms((name,))
        out[f"without_{name}_ms"] = round(ms, 4)
        out[f"{name}_us_per_layer"] = round((full - ms) * 1e3 / eng.L, 2)
    ms = graph_ms(("rope", "attn", "norm", "swiglu"))
    out["gemms_only_ms"] = round(ms, 4)
    out["gemms_only_us_per_layer"] = round(ms * 1e3 / eng.L, 2)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
