"""Record the UNMODIFIED reference's side of the GPU parity tests (tests/test_gpu_vs_reference.py) -> parity_ref.json.gz.

Needs a CUDA device and the reference (``LADE_REFERENCE_ROOT`` or ``baseline/_ref``, see baseline/ref_loader.py).  For every
case of the parity tests it runs the reference's own ``jacobi_greedy_search_multilevel`` on the GPU, with the weights the
tests build (bench.build_model, seeded on the device), and stores

  * its token ids and step count;
  * for every generated position, the top-4 next-token logits of the reference model's own teacher-forced causal forward
    over its ids (the logits a divergence is judged on, baseline/parity.py);
  * the reference's self-consistency on the run (the width of a tie on this model).

    LADE_REFERENCE_ROOT=<reference checkout> python tests/golden/gen_golden_parity.py
"""
import gzip
import json
import os
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path[:0] = [ROOT, os.path.dirname(HERE)]

from baseline import parity as PAR  # noqa: E402
import test_gpu_vs_reference as T  # noqa: E402

TOPK = 4


def record(ref, ids, n_prompt, steps=None):
    dev = next(ref.parameters()).device
    with PAR._reference_device(dev, next(ref.parameters()).dtype), torch.no_grad():
        x = torch.tensor([ids[:-1]], dtype=torch.long, device=dev)
        out = ref.model.LlamaModeljforward(input_ids=x, is_prefill=True, level_sizes=[x.size(1) - 1], guess=None,
                                           use_cache=False)
        h = out[0] if isinstance(out, tuple) else out.last_hidden_state
        logits = ref.lm_head(h[0, n_prompt - 1:, :]).float()
    top = torch.topk(logits, TOPK, dim=-1)
    return {"ids": list(ids), "n_prompt": n_prompt, "steps": steps, "topk_ids": top.indices.tolist(),
            "topk_logits": top.values.tolist(), "self": PAR.reference_self_consistency(ref, ids, n_prompt)}


def prompt_of(shape, P, seed=1):
    g = torch.Generator().manual_seed(seed)
    return torch.randint(3, shape["vocab"], (P,), generator=g).tolist()


def main():
    assert torch.cuda.is_available()
    torch.cuda.set_device(0)
    gold = {"gpu": torch.cuda.get_device_name(0)}
    fp16 = {c[0] for c in T.CASES if c[0] in T.FP16_CASES}
    for name, shape, W, N, G, P, new, pool in T.CASES:
        for dt in (torch.bfloat16, torch.float16) if name in fp16 else (torch.bfloat16,):
            hf, ref = T.build_pair(shape, dtype=dt)
            prompt = prompt_of(shape, P)
            ids, steps = PAR.reference_greedy(ref, prompt, new, W, N, G, py_seed=0, pool_from_prompt=pool)
            gold[name if dt == torch.bfloat16 else name + "_fp16"] = record(ref, ids, P, steps)
            print(name, dt, steps, flush=True)
            del hf, ref
    # EOS on the first token (W5 N3 G3, pool from the prompt)
    hf, ref = T.build_pair(T.TINY)
    prompt = prompt_of(T.TINY, 12)
    free, _ = PAR.reference_greedy(ref, prompt, 16, 5, 3, 3, py_seed=0, pool_from_prompt=True)
    eos = free[12]
    ids, steps = PAR.reference_greedy(ref, prompt, 16, 5, 3, 3, py_seed=0, eos_token_id=[eos], pool_from_prompt=True)
    gold["eos_first_token"] = dict(record(ref, ids, 12, steps), eos=eos)
    # the reference model's plain greedy (its causal forward, argmax) after a 10-token prompt
    prompt = prompt_of(T.TINY, 10, seed=3)
    ar = list(prompt)
    for _ in range(24):
        ar.append(int(torch.argmax(PAR.reference_next_logits(ref, ar))))
    gold["plain_greedy_p10"] = record(ref, ar, 10)
    with gzip.open(os.path.join(HERE, "parity_ref.json.gz"), "wt") as f:
        json.dump(gold, f, separators=(",", ":"))
    print("wrote", os.path.join(HERE, "parity_ref.json.gz"))


if __name__ == "__main__":
    main()
