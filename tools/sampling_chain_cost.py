"""Device time of the sampling verification kernel (lade_sample_verify, bf16) on two workloads:

* bench: the benchmark's sampling configuration, V 32000, W 15 / N 5 / G 15, T 0.8, on rows where the first n-grams
  are rejected and a later one accepted (a few rejections per position, then the residual draw);
* deep: V 152064, G 1024 / N 3, one position with 1000 rejected candidates holding 1 - 1e-4 of the mass, then the
  residual draw.

Each library given with --lib is timed in its own process (CUDA events around --iters launches, median of --reps),
the processes alternating --rounds times so that drift on a shared host hits both alike.  Prints one JSON line per
(library, round) and a summary line with the GPU name and power limit.

    python tools/sampling_chain_cost.py --lib lookaheaddecoding_b200/lib/liblade_sm100.so [--lib other.so]"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def worker(lib_path, iters, reps):
    sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]
    import numpy as np
    import torch
    from lookaheaddecoding_b200 import _cabi
    _cabi._build.LIB_PATH = os.path.abspath(lib_path)
    _cabi.load(build_if_missing=False)
    from sampling_ctx import Bare, device_logits

    out = {}
    rng = np.random.default_rng(0)
    # bench: 15 n-grams of GS 4, candidates at position 0 drawn from the row's top tokens
    h = Bare(15, 5, 15)
    V = 32000
    rows = rng.normal(0, 2.0, (h.n_rows, V))
    top = rng.choice(V, 8, replace=False)
    rows[:, top] += np.linspace(6.0, 4.0, 8)
    logits = device_logits(torch.bfloat16, rows, V, 0.0)
    guess = [int(top[e % 8]) if i == 0 else int(top[(e + i) % 8]) for e in range(15) for i in range(4)]
    meta = h.set_guess(guess)
    out["bench"] = _time(h, logits, V, meta, 0.8, iters, reps)
    h.close()
    # deep: 1000 rejections at one position
    h = Bare(20, 3, 1024)
    V = 152064
    p = np.full(V, 1e-4 / V)
    cands = rng.choice(V, 1001, replace=False)
    p[cands[:1000]] = (1 - 1e-4) / 1000
    logits = device_logits(torch.bfloat16, np.log(p), V, 0.0).expand(h.n_rows, -1).contiguous()
    guess = [int(t) for c in cands for t in (c, 5)]
    meta = h.set_guess(guess[:2 * 1001])
    # offsets whose first 1000 uniforms all reject (u > 1/1000 - ... : conditional p_j = 1 / (1000 - j) roughly)
    from oracle import philox as PX
    u = PX.uniforms(3, 0, 1 << 22).astype(np.float64)
    pj = np.array([1.0 / (1000 - j + 1e-4 * 1000) for j in range(1000)])
    idx = np.arange((1 << 22) - 1100)
    for j in range(1000):
        idx = idx[u[idx + j] > pj[j] * 1.01]
        if not len(idx):
            break
    if len(idx):
        out["deep"] = _time(h, logits, V, meta, 1.0, max(1, iters // 10), reps, offset=int(idx[0]))
    else:
        print("warning: no offset in the scanned stream rejects all 1000 candidates; deep workload not timed",
              file=sys.stderr)
    h.close()
    print(json.dumps(out))


def _time(h, logits, V, meta, T, iters, reps, offset=0):
    import torch
    for _ in range(5):                         # Bare.launch checks the return code
        h.launch(torch.bfloat16, logits, V, meta, T, seed=1, offset=offset, dbg=False)
    h.launch(torch.bfloat16, logits, V, meta, T, seed=1, offset=offset)
    n_draws = len(h.exported())
    times = []
    fn = h.lib.lade_sample_verify
    rec = torch.zeros(h.REC, dtype=torch.int32, device="cuda")
    rng0 = torch.tensor([1, offset], dtype=torch.int64, device="cuda")
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        rcs = set()
        for _ in range(iters):
            h.rng.copy_(rng0)                  # every launch replays the same chain
            rc = fn(h.ctx, h.stream, logits.data_ptr(), logits.shape[1], V, h.am.data_ptr(), meta.data_ptr(),
                    float(T), 0, 1.0, h.rng.data_ptr(), rec.data_ptr(), 0)
            rcs.add(rc)
        b.record()
        torch.cuda.synchronize()
        if rcs != {0}:
            raise RuntimeError(f"lade_sample_verify returned {sorted(rcs)}")
        times.append(a.elapsed_time(b) * 1000.0 / iters)
    times.sort()
    return {"us_median": round(times[len(times) // 2], 2), "us_min": round(times[0], 2), "draws": n_draws}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lib", action="append", required=True)
    ap.add_argument("--iters", type=int, default=2000)
    ap.add_argument("--reps", type=int, default=9)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--worker", action="store_true")
    a = ap.parse_args()
    if a.worker:
        return worker(a.lib[0], a.iters, a.reps)
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    res = {lib: [] for lib in a.lib}
    for r in range(a.rounds):
        for lib in a.lib:
            p = subprocess.run([sys.executable, __file__, "--worker", "--lib", lib, "--iters", str(a.iters),
                                "--reps", str(a.reps)], capture_output=True, text=True)
            if p.returncode:
                sys.exit(p.stderr)
            for warn in (ln for ln in p.stderr.splitlines() if ln.startswith("warning:")):
                print(warn, file=sys.stderr)
            line = json.loads(p.stdout.strip().splitlines()[-1])
            res[lib].append(line)
            print(json.dumps({"lib": lib, "round": r, **line}))
    print(json.dumps({"gpu": gpu, "summary": {lib: {k: sorted(x[k]["us_median"] for x in v if k in x)
                                                   for k in ("bench", "deep")} for lib, v in res.items()}}))


if __name__ == "__main__":
    main()
