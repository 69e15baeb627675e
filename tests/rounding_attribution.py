#!/usr/bin/env python
"""CHECKER (not a test, not product): which rounding-order differences explain the token-id divergences from the
unmodified reference at the Llama-2-7B shape with random weights?

The engine differs from the reference's CUDA-eager run in two places that change the ORDER of roundings (never the
rounding points of the scores): (a) the lookahead-attention kernel rounds the unnormalised probabilities to the model
dtype and normalises the fp32 result (online softmax), the reference normalises in fp32 and rounds after
(modeling_llama.py:520-541); (b) q/k/v and gate/up run as ONE library GEMM each instead of three / two, which may pick
another cuBLAS kernel (other accumulation order).  This script re-runs the id comparison of baseline/parity.py with
either difference removed by replacing a stage method on its own engine instance:

  A  engine as shipped
  B  projections issued call for call like the reference (engine._proj replaced)
  C  attention replaced by the restated reference math in torch on the engine's own Q / KV cache (engine._attention)
  D  B + C
  E  the engine with attn_impl=3: the wgmma kernel's reference-order variant (no stage replaced, CUDA graph on)

and prints one JSON line with the number of divergences of each against the reference's own self-inconsistency on the
same run (ids of its lookahead loop vs its own teacher-forced forward).  usage (GPU box):
    python tests/rounding_attribution.py [--max-new 128] [--prompt-len 1024]
"""
import argparse
import json
import os
import random
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

from lookaheaddecoding_b200 import LookaheadEngine, _cabi  # noqa: E402
from oracle import llama_ref as LR  # noqa: E402


def unfused_proj(eng):
    """engine._proj, with the fused q/k/v and gate/up weights (recognised by identity) issued call for call like the
    reference (modeling_llama.py:447-449,:378)."""
    nq, nk = eng.nh * eng.D, eng.nkv * eng.D
    parts = {id(w): (nq, nk, nk) for w in eng.w_qkv}
    parts.update({id(w): (eng.I, eng.I) for w in eng.w_gu})

    def proj(x, w, out):
        if id(w) not in parts:
            return LookaheadEngine._proj(eng, x, w, out)
        for w_part, out_part in zip(w.split(parts[id(w)]), out.split(parts[id(w)], dim=1)):
            torch.mm(x, w_part.t(), out=out_part)
        return 0
    return proj


def reference_attention(eng):
    """engine._attention, restated in torch (runs without a CUDA graph: reads the step's geometry on the host)."""
    geom = {}

    def attention(stream, l, qb, kc, vc, attn_out, rows, prefill):
        if l == 0:     # one host read of the step's geometry per step
            meta = eng.meta.cpu()
            q_len, kv_len = int(meta[_cabi.M_Q_LEN]), int(meta[_cabi.M_KV_LEN])
            if prefill:
                vis = torch.tril(torch.ones(q_len, q_len, dtype=torch.bool, device=eng.dev))
            else:
                mw = eng.mask_words          # flat [rows][mw] uint32 words, bit c of row r = step column c visible
                words = eng.rowmask[: q_len * mw].cpu().numpy().view(np.uint32).reshape(q_len, mw)
                bits = np.unpackbits(words.view(np.uint8), axis=-1, bitorder="little")[:, :q_len].astype(bool)
                vis = torch.from_numpy(bits).to(eng.dev)
            geom["step"] = (q_len, kv_len, LR.additive_mask(vis, kv_len, eng.dt))
        q_len, kv_len, mask = geom["step"]
        T = kv_len + q_len
        o = LR.eager_attention(qb[:, :q_len], kc[:, :T], vc[:, :T], mask, eng.nh // eng.nkv)
        attn_out[:q_len] = o.transpose(0, 1).reshape(q_len, -1)
        return 0
    return attention


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--max-new", type=int, default=128)
    ap.add_argument("--prompt-len", type=int, default=1024)
    ap.add_argument("--modes", default="A,B,C,D,E")
    args = ap.parse_args()

    import bench
    from baseline import parity as PAR

    shape, W, N, G, _ = bench.WORKLOADS["7b"]
    P = args.prompt_len
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    model = bench.build_model(shape, dev)
    torch.manual_seed(1)
    prompt = torch.randint(3, shape["vocab"], (P,)).tolist()

    ref_model = PAR.reference_model_sharing_weights(model, shape)
    ref_ids, _ = PAR.reference_greedy(ref_model, prompt, args.max_new, W, N, G, py_seed=0)
    self_rep = PAR.reference_self_consistency(ref_model, ref_ids, P)
    out = {"compared_tokens": args.max_new, "prompt_len": P,
           "reference_self_mismatches": self_rep["n_self_mismatch"], "modes": {}}
    names = {"A": "as shipped", "B": "projections call for call", "C": "reference-order attention (torch)",
             "D": "both", "E": "attn_impl=3 (reference-order wgmma kernel)"}
    for mode in args.modes.split(","):
        eng = LookaheadEngine(model, W, N, G, pool_from_prompt=True, max_total_len=P + args.max_new + 8,
                              use_cuda_graph=mode in ("A", "B", "E"), attn_impl=3 if mode == "E" else 0)
        if mode in ("B", "D"):
            eng._proj = unfused_proj(eng)
        if mode in ("C", "D"):
            eng._attention = reference_attention(eng)
        rep = PAR.compare_ids(lambda p_, n_: eng.generate(p_, n_, rng=random.Random(0)), ref_ids, P, ref_model,
                              self_check=False, max_divergences=args.max_new)
        out["modes"][mode] = {"what": names[mode], "n_divergences": rep["n_divergences"],
                              "exact_prefix_tokens": rep["exact_prefix_tokens"],
                              "worst_candidate_below_top_ulps": rep["worst_candidate_below_top_ulps"]}
        eng.close()
        del eng
        torch.cuda.empty_cache()
        print(json.dumps({mode: out["modes"][mode]}), file=sys.stderr, flush=True)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
