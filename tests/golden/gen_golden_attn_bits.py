#!/usr/bin/env python
"""Bit-exact fingerprints of the wgmma attention kernel (impl 2 and its reference-order variant, impl 3).

Writes tests/golden/attn_bits.json: for every case below, the SHA-256 of the bytes lade_attn_fwd(_f16) writes for
inputs drawn from a seeded CPU torch.Generator.  Rescheduling the kernel (launch shape, split merge, pipelining) must not
change a single output bit, and tests/test_gpu_attention_bits.py holds later builds to these hashes.  Run once on an
H100 with the library whose outputs are the reference:

    python tests/golden/gen_golden_attn_bits.py [OUT.json]
"""
import hashlib
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from oracle import lookahead as LA  # noqa: E402

OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "attn_bits.json")
D = 128

# name: (kind, shape, kv_len, Hq, Hkv, n_splits, extra q_pad rows, impls)
#   kind "steady": the single-GPU lookahead step of (W, N, G); "prefill": P causal rows; "lp": rank 1 of 4 under lookahead
#   parallelism (re-fed tokens and a foreign level-0 prefix: level and dist offsets)
CASES = {
    "bench_kv1024_s4": ("steady", (15, 5, 15), 1024, 32, 32, 4, 0, (2, 3)),
    "bench_kv1278_s4": ("steady", (15, 5, 15), 1278, 32, 32, 4, 0, (2, 3)),
    "13b_h40_s3": ("steady", (20, 7, 20), 517, 40, 40, 3, 0, (2, 3)),       # 240 rows: two q tiles
    "splits1": ("steady", (15, 5, 15), 200, 4, 4, 1, 4, (2, 3)),
    "splits3": ("steady", (15, 5, 15), 700, 4, 4, 3, 4, (2, 3)),
    "splits5": ("steady", (15, 5, 15), 1000, 4, 4, 5, 0, (2, 3)),
    "ring_wrap_s3": ("steady", (15, 5, 15), 3001, 2, 2, 3, 0, (2,)),          # > 3 K/V tiles per split
    "gqa_h8_kv2_s4": ("steady", (15, 5, 15), 900, 8, 2, 4, 0, (2, 3)),
    "prefill_300_s3": ("prefill", (300,), 0, 2, 2, 3, 0, (2, 3)),             # three q tiles
    "lp_offset_s2": ("lp", (15, 5, 2), 77, 2, 2, 2, 0, (2, 3)),
    "q16_s4": ("steady", (5, 3, 3), 200, 4, 4, 4, 0, (2, 3)),                 # q <= 64: one warpgroup idles
}
DTYPES = {"bf16": torch.bfloat16, "fp16": torch.float16}


def layout(kind, shape):
    if kind == "steady":
        W, N, G = shape
        gs = N - 1
        return LA.layout_from_shape([W - 1] + [W] * (N - 2), 1, G * gs, gs)
    if kind == "prefill":
        (P,) = shape
        return LA.layout_from_shape([P - 1], 1, 0, 4, is_prefill=True)
    W, N, g = shape
    gs, workers, skip, r = N - 1, 4, 2, 1
    split = (W + workers - 1) // workers
    ws, we = min(split * r, W), min(split * (r + 1), W)
    return LA.layout_from_shape([we - 1] + [we - ws] * (N - 2), 1 + skip, g * gs, gs)


def run_case(name, impl, dtype_name):
    """SHA-256 of the kernel's output rows [0, q_pad) for case `name`."""
    from lookaheaddecoding_b200 import _cabi
    lib = _cabi.load()
    kind, shape, kv_len, Hq, Hkv, n_splits, pad, _ = CASES[name]
    dt = DTYPES[dtype_name]
    lay = layout(kind, shape)
    q_len = lay.q_len
    q_pad = q_len + pad
    T = kv_len + q_len
    cap = T + 70
    g = torch.Generator().manual_seed(sum(map(ord, name)))
    qb = torch.zeros(Hq, q_pad, D, dtype=dt)
    qb[:, :q_len] = torch.randn(Hq, q_len, D, generator=g).to(dt)
    kc = torch.full((Hkv, cap, D), float("nan"), dtype=dt)          # stale cache rows must never reach the output
    vc = torch.full((Hkv, cap, D), float("nan"), dtype=dt)
    kc[:, :T] = torch.randn(Hkv, T, D, generator=g).to(dt)
    vc[:, :T] = torch.randn(Hkv, T, D, generator=g).to(dt)
    qb, kc, vc = qb.cuda(), kc.cuda(), vc.cuda()
    out = torch.zeros(q_pad, Hq * D, dtype=dt, device="cuda")
    meta = torch.zeros(_cabi.META_INTS, dtype=torch.int32, device="cuda")
    for key, val in {_cabi.M_Q_LEN: q_len, _cabi.M_KV_LEN: kv_len, _cabi.M_N_INPUT: lay.n_input,
                     _cabi.M_LEVEL_OFFSET: lay.level_offset, _cabi.M_ALL_OFFSET: lay.level_offset + lay.dist_offset,
                     _cabi.M_TINY: lay.tiny, _cabi.M_N_LEVELS: len(lay.level_sizes), _cabi.M_N_GUESS_TOK: lay.n_guess_tok,
                     _cabi.M_IS_PREFILL: int(lay.is_prefill), _cabi.M_Q_PAD: q_pad}.items():
        meta[key] = val
    mw = (q_pad + 31) // 32 + 1
    bits = np.zeros((q_pad, mw * 32), dtype=bool)
    if not lay.is_prefill:
        bits[:q_len, :q_len] = LA.step_mask(lay)
    words = np.packbits(bits.reshape(q_pad, mw, 32), axis=-1, bitorder="little").view(np.uint32).reshape(q_pad, mw)
    rowmask = torch.from_numpy(words.view(np.int32).copy()).cuda()
    scratch = torch.zeros(lib.lade_attn_scratch_bytes(q_pad, Hq, D, n_splits), dtype=torch.uint8, device="cuda")
    fwd = lib.lade_attn_fwd if dt == torch.bfloat16 else lib.lade_attn_fwd_f16
    _cabi.check(fwd(torch.cuda.current_stream().cuda_stream, qb.data_ptr(), kc.data_ptr(), vc.data_ptr(), out.data_ptr(),
                    0 if lay.is_prefill else rowmask.data_ptr(), mw, meta.data_ptr(), scratch.data_ptr(), q_pad, Hq, Hkv,
                    D, cap, T, n_splits, impl), "lade_attn_fwd")
    torch.cuda.synchronize()
    assert int(scratch[:65536].view(torch.int32).abs().sum()) == 0, "split counters must self-reset"
    return hashlib.sha256(out.cpu().contiguous().view(torch.uint8).numpy().tobytes()).hexdigest()


def keys():
    for name, case in CASES.items():
        for impl in case[7]:
            for dtn in DTYPES:
                yield name, impl, dtn


def main():
    out_path = sys.argv[1] if len(sys.argv) > 1 else OUT
    hashes = {f"{n}/impl{i}/{d}": run_case(n, i, d) for n, i, d in keys()}
    rec = {"gpu": torch.cuda.get_device_name(0), "sha256": hashes}
    with open(out_path, "w") as f:
        json.dump(rec, f, indent=1, sort_keys=True)
    print(f"{len(hashes)} hashes -> {out_path}")


if __name__ == "__main__":
    main()
