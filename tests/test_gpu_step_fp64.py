"""Every row of the engine's lookahead step held to a float64 forward of the same model, step by step.

The id tests (test_gpu_e2e, test_gpu_vs_reference, test_gpu_qwen3) cannot see most of a lookahead step: decoding is
lossless, so a window row computed wrong only lowers the acceptance, and a KV row compacted from the wrong source moves
later logits by little on a random-init model.  Here the engine is driven in lockstep with the oracle's lookahead loop
(oracle.lookahead.greedy_lookahead, the same prompt and initial-window draws as engine.draw_window) and, at every step:

* the engine's step rows (ids, positions) equal the oracle layout's;
* the same layout, with the oracle's own mask (LA.step_mask, not the device's rowmask), runs through two OracleLlama:
  float64 (the truth; RoPE tables of the model dtype widened, the operands the engine uses) and the model dtype (an
  honest model-dtype pipeline, the yardstick);
* logits at every used lm slot (slot 0, the window slots, the guess slots) against the float64 logits of the row the
  oracle says that slot stands for: with e_eng = engine - f64 and e_ref = model-dtype oracle - f64 over the vocabulary,
  rms(e_eng) <= R rms(e_ref) + ulp(rms|f64|) / 16 and max|e_eng| <= R max|e_ref| + ulp(max|f64|);
* the KV cache after the step's compaction, per layer, K / V and KV head, by the same ratio test against the float64
  oracle's post-norm, post-RoPE cache (prompt rows, each step's input row, every compacted guess row);
* am[s] is a token whose float64 logit is within 2 max|e_eng| of that slot's float64 maximum;
* with a second engine that replays the steady step from a CUDA graph: logits, am and the KV cache bit-identical.

The engine's own am tokens drive the oracle's state, so the two never drift apart on a tie.

Planted faults, each on an eager engine by wrapping a stage method or editing pos / rowmask / lm_rows / res after the
layout, must fail these checks; the first three keep the ids within the existing tie allowance (assert_same_or_tie),
which is why the id tests cannot see them.
"""
import functools
import random

import pytest
import torch

from oracle import llama_ref as LR
from oracle import lookahead as LA

pytestmark = pytest.mark.gpu

LLAMA = dict(hidden=256, layers=2, heads=2, kv_heads=2, inter=688, vocab=32000, max_pos=2048, rope_theta=10000.0, eps=1e-5)
GQA = dict(hidden=512, layers=2, heads=4, kv_heads=2, inter=688, vocab=4096, max_pos=2048, rope_theta=10000.0, eps=1e-5)
D64 = dict(hidden=256, layers=2, heads=4, kv_heads=2, inter=688, vocab=4096, max_pos=2048, rope_theta=10000.0, eps=1e-5)
PERIODIC = dict(hidden=256, layers=2, heads=2, kv_heads=2, inter=688, vocab=4096, max_pos=2048, rope_theta=10000.0,
                eps=1e-5)
# "periodic with attention": bench.build_model(weights="cyclic") makes the next token a function of the last one (every
# layer is the identity on the residual stream), so n-grams repeat and guesses are accepted.  o_proj gets a small random
# weight, normal(0, O_SCALE): attention then moves the logits (about 7 % rms of their size), while the periodic next
# token still wins almost everywhere.  lm_head is scaled as in test_gpu_sampling_device.peaked_periodic_model.
O_SCALE, LM_SCALE = 0.001, 30.0

#          name              model        dtype            W   N  G   P    new  attn graph
CASES = {"llama_mha":      ("llama", LLAMA, torch.bfloat16, 15, 5, 15, 32, 48, 0, True),
         "llama_gqa":      ("llama", GQA, torch.bfloat16, 15, 5, 15, 32, 48, 0, False),
         "llama_d64":      ("llama", D64, torch.bfloat16, 7, 4, 7, 32, 48, 0, False),
         "periodic_bf16":  ("periodic", PERIODIC, torch.bfloat16, 7, 4, 7, 24, 160, 0, True),
         "periodic_fp16":  ("periodic", PERIODIC, torch.float16, 7, 4, 7, 24, 160, 0, True),
         # several prefill query tiles; N = 3 has no window-fill step
         "llama_prompt300": ("llama", LLAMA, torch.bfloat16, 5, 3, 3, 300, 32, 0, False),
         # several window-fill steps, a larger step
         "llama_w20n7g20": ("llama", LLAMA, torch.bfloat16, 20, 7, 20, 48, 48, 0, False),
         # heads * head_dim != hidden, vocab 151936; the default attention and the reference-order one
         "qwen3_impl0":    ("qwen3", None, torch.bfloat16, 15, 5, 15, 32, 48, 0, False),
         "qwen3_impl3":    ("qwen3", None, torch.bfloat16, 15, 5, 15, 32, 48, 3, False)}

# The ratio bound R per model family.  Worst honest ratios measured on an H100 SXM (700 W), over every step, slot, layer
# and head (rms / max): Llama 1.32 / 1.59 (KV 1.01 / 1.33), periodic 1.10 / 1.58 (KV 1.01 / 1.07), Qwen3 1.50 / 1.58 with
# attn_impl 0 and 1.06 / 1.15 with attn_impl 3 (KV 1.00 / 1.18).  The weakest planted fault (one extra visible mask
# column) reaches 8.8.
R_BOUND = {"llama": 2.5, "periodic": 2.5, "qwen3": 2.5}
# At least this many steps with an accepted guess, and with a full accept, on the periodic model.  A full accept is
# max_hit == N - 2: the reference's verification loop (decoding.py:1071-1084, oracle.lookahead.verify_guesses) never
# reports more, and lade_kv_compact moves at most N - 2 rows.  Measured on an H100 over 160 new tokens: bf16 112 steps,
# 25 with an accept, 23 full; fp16 99 steps, 31 with an accept, 31 full.
MIN_ACCEPT_STEPS, MIN_FULL_ACCEPTS = 10, 5


@functools.lru_cache(maxsize=1)
def build(name):
    """(HF model, oracle cfg, weights) of case `name` (one model alive at a time)."""
    kind, shape, dtype = CASES[name][:3]
    if kind == "qwen3":
        from test_gpu_qwen3 import build_qwen3
        model = build_qwen3(head_dim=128, tie=False, dtype=dtype)
    else:
        from bench import build_model
        model = build_model(shape, torch.device("cuda"), seed=0, weights="cyclic" if kind == "periodic" else "random",
                            dtype=dtype)
        if kind == "periodic":
            g = torch.Generator(device="cuda").manual_seed(11)
            with torch.no_grad():
                model.lm_head.weight.mul_(LM_SCALE)
                for layer in model.model.layers:
                    layer.self_attn.o_proj.weight.normal_(0.0, O_SCALE, generator=g)
    c = model.config
    ocfg = dict(hidden=c.hidden_size, layers=c.num_hidden_layers, heads=c.num_attention_heads,
                kv_heads=c.num_key_value_heads, inter=c.intermediate_size, vocab=c.vocab_size,
                max_pos=c.max_position_embeddings, eps=c.rms_norm_eps, rope_theta=c.rope_parameters["rope_theta"],
                head_dim=getattr(c, "head_dim", None) or c.hidden_size // c.num_attention_heads)
    w = {k: v.detach().clone() for k, v in model.state_dict().items() if "rotary" not in k}
    return model, ocfg, w


def prompt_of(name):
    shape_vocab = CASES[name][1]["vocab"] if CASES[name][1] else 151936
    return torch.randint(3, shape_vocab, (CASES[name][6],), generator=torch.Generator().manual_seed(1)).tolist()


def make_engine(name, **kw):
    from lookaheaddecoding_b200 import LookaheadEngine
    _, _, _, W, N, G, P, new, attn, _ = CASES[name]
    model = build(name)[0]
    return LookaheadEngine(model, W, N, G, pool_from_prompt=True, max_total_len=P + new, attn_impl=attn, **kw)


def _ulp(x: torch.Tensor, dtype) -> torch.Tensor:
    return LR.ulp(x, dtype)


def ratio_check(got, ref, md, R, dtype, dims):
    """(ok per group, rms ratio, max ratio) of got / md against ref (all float64), reduced over `dims`."""
    e_eng, e_ref = got - ref, md - ref
    rms = lambda e: e.pow(2).mean(dims).sqrt()          # noqa: E731
    mx = lambda e: e.abs().amax(dims)                  # noqa: E731
    r_eng, r_ref, m_eng, m_ref = rms(e_eng), rms(e_ref), mx(e_eng), mx(e_ref)
    ok = (r_eng <= R * r_ref + _ulp(rms(ref), dtype) / 16) & (m_eng <= R * m_ref + _ulp(mx(ref), dtype))
    tiny = torch.finfo(torch.float64).tiny
    return ok, r_eng / r_ref.clamp_min(tiny), m_eng / m_ref.clamp_min(tiny), m_eng


class Report:
    def __init__(self, name):
        self.name = name
        self.steps = self.accept_steps = self.full_accepts = 0
        self.logit_rms = self.logit_max = self.kv_rms = self.kv_max = 0.0
        self.failures = []          # (step, check, detail)
        self.graph_diffs = []

    def fail(self, step, check, detail):
        self.failures.append((step, check, detail))

    def kinds(self):
        return {f[1] for f in self.failures}

    def line(self):
        return (f"{self.name}: {self.steps} steps, {self.accept_steps} with an accept, {self.full_accepts} full; worst "
                f"ratio logits rms {self.logit_rms:.2f} max {self.logit_max:.2f}, KV rms {self.kv_rms:.2f} max "
                f"{self.kv_max:.2f}; {len(self.failures)} failed checks {sorted(self.kinds())}")


@torch.no_grad()
def run_lockstep(name, engines, R=None):
    """Drive `engines` (the first is checked against the oracles, any other must match it bit for bit) with the
    oracle's lookahead loop over case `name`; returns the Report."""
    from lookaheaddecoding_b200 import _cabi
    kind, _, dtype, W, N, G, P, new, _, _ = CASES[name]
    R = R_BOUND[kind] if R is None else R
    model, ocfg, w = build(name)
    # the float64 oracle widens the embedding rows it gathers and lm_head chunk by chunk (no float64 copy of either)
    narrow = ("model.embed_tokens.weight", "lm_head.weight")
    o64 = LR.OracleLlama(ocfg, {k: v if k in narrow else v.double() for k, v in w.items()}, device="cuda",
                         rope_dtype=dtype)
    omd = LR.OracleLlama(ocfg, w, device="cuda")
    prompt = prompt_of(name)
    WCAP, GS = W + N - 3, N - 1
    rep = Report(name)
    eng = engines[0]
    window0 = eng.draw_window(prompt, random.Random(5))
    for e in engines:
        e.begin(prompt, P + new, (), window0)
    st = {"step": 0}

    def step_fn(lay, kv_len):
        i = st["step"]
        for e in engines:
            e.run_forward_step(i, P)
        torch.cuda.synchronize()
        meta = eng.meta.cpu().tolist()
        q = lay.q_len
        assert meta[_cabi.M_Q_LEN] == q and meta[_cabi.M_KV_LEN] == kv_len, (name, i)
        if eng.ids[:q].cpu().tolist() != lay.ids or eng.pos[:q].cpu().tolist() != lay.pos:
            rep.fail(i, "layout", "step rows differ from the oracle layout's ids / positions")
        vis = torch.from_numpy(LA.step_mask(lay))
        lg, tiny = lay.n_guess_tok, lay.level_sizes[-1]
        slots = [0] + [1 + j for j in range(tiny)] + [1 + WCAP + j for j in range(lg)]
        rows = [lay.n_input - 1] + [q - lg - tiny + j for j in range(tiny)] + [q - lg + j for j in range(lg)]
        ref = o64.forward_rows(lay.ids, lay.pos, vis, kv_len, logit_rows=rows)
        mdr = omd.forward_rows(lay.ids, lay.pos, vis, kv_len, logit_rows=rows).double()
        got = eng.logits[slots].double()
        ok, r_rms, r_max, m_eng = ratio_check(got, ref, mdr, R, dtype, dims=-1)
        rep.logit_rms, rep.logit_max = max(rep.logit_rms, r_rms.max().item()), max(rep.logit_max, r_max.max().item())
        for k in (~ok).nonzero().flatten().tolist():
            rep.fail(i, "logits", f"slot {slots[k]} row {rows[k]}: rms ratio {r_rms[k]:.2f} max ratio {r_max[k]:.2f}")
        am = eng.am.cpu()
        top = ref.max(-1).values
        chosen = ref.gather(1, am[slots].long().cuda()[:, None])[:, 0]
        bad = top - chosen > 2 * m_eng
        for k in bad.nonzero().flatten().tolist():
            rep.fail(i, "argmax", f"slot {slots[k]}: am {int(am[slots[k]])} is {top[k] - chosen[k]:.4g} below the top")
        for e in engines[1:]:
            if not (torch.equal(e.logits, eng.logits) and torch.equal(e.am, eng.am)):
                rep.graph_diffs.append((i, "logits/am"))
        st["step"] = i + 1
        rep.steps += 1
        am = am.tolist()
        return am[0], am[1:1 + tiny], am[1 + WCAP:1 + WCAP + lg]

    def compact_fn(dst, src, n, new_len):
        i = st["step"] - 1
        for o in (o64, omd):
            o.compact_fn(dst, src, n, new_len)
        if n > 0:
            rep.accept_steps += 1
            rep.full_accepts += int(n == N - 2)
        res = eng.res.cpu().tolist()
        assert res[_cabi.R_KV_LEN] == new_len and res[_cabi.R_MAX_HIT] == n, (name, i)
        for l in range(ocfg["layers"]):
            got = eng.kv[l, :, :, :new_len].double()                       # [2, nkv, new_len, D]
            ref = torch.stack([o64.k_cache[l], o64.v_cache[l]])
            mdc = torch.stack([omd.k_cache[l], omd.v_cache[l]]).double()
            ok, r_rms, r_max, _ = ratio_check(got, ref, mdc, R, dtype, dims=(-2, -1))
            rep.kv_rms, rep.kv_max = max(rep.kv_rms, r_rms.max().item()), max(rep.kv_max, r_max.max().item())
            for t, h in (~ok).nonzero().tolist():
                rep.fail(i, "kv", f"layer {l} {'KV'[t]} head {h}: rms ratio {r_rms[t, h]:.2f} max ratio "
                                  f"{r_max[t, h]:.2f}")
            for e in engines[1:]:
                if not torch.equal(e.kv[l, :, :, :new_len], eng.kv[l, :, :, :new_len]):
                    rep.graph_diffs.append((i, f"kv layer {l}"))

    ids, steps = LA.greedy_lookahead(prompt, new, W, N, G, step_fn, compact_fn, pool_from_prompt=True,
                                     rng=random.Random(5))
    assert steps == rep.steps
    return rep


HONEST = {}


@pytest.mark.parametrize("name", list(CASES))
def test_step_rows_match_float64(name):
    graph = CASES[name][9]
    engines = [make_engine(name, use_cuda_graph=True), make_engine(name, use_cuda_graph=False)] if graph else \
        [make_engine(name, use_cuda_graph=False)]
    rep = run_lockstep(name, engines)
    HONEST[name] = rep
    print("\n" + rep.line() + (f"; graph vs eager: {len(rep.graph_diffs)} differences" if graph else ""))
    for f in rep.failures[:10]:
        print("   ", f)
    assert not rep.failures, rep.failures[:10]
    assert not rep.graph_diffs, rep.graph_diffs[:10]
    if CASES[name][0] == "periodic":
        assert rep.accept_steps >= MIN_ACCEPT_STEPS and rep.full_accepts >= MIN_FULL_ACCEPTS, rep.line()
    for e in engines:
        e.close()


# ---- planted faults -------------------------------------------------------------------------------------------------
def _layout_now(eng):
    from lookaheaddecoding_b200 import _cabi
    m = eng.meta.cpu().tolist()
    return dict(q=m[_cabi.M_Q_LEN], kv=m[_cabi.M_KV_LEN], n_input=m[_cabi.M_N_INPUT], tiny=m[_cabi.M_TINY],
                lg=m[_cabi.M_N_GUESS_TOK], prefill=bool(m[_cabi.M_IS_PREFILL]))


def plant(eng, fault):
    """Plant `fault` on the eager engine `eng` (edits after the step's layout, at layer 0's RoPE stage, or a
    replaced commit).  Every edit stays inside the buffers the step already uses."""
    from lookaheaddecoding_b200 import _cabi
    from lookaheaddecoding_b200._cabi import check
    from lookaheaddecoding_b200.engine import _ptr
    assert not eng.use_cuda_graph
    rope = eng._rope_append

    def rope_after_layout(stream, l, *a):
        if l == 0:
            lay = _layout_now(eng)
            last_level0 = lay["q"] - lay["lg"] - lay["tiny"]               # first window row of the last level
            if fault == "mask" and not lay["prefill"]:
                mw = eng.mask_words
                r = lay["q"] - lay["lg"] - 1                                 # last window row of the last level
                words = eng.rowmask[r * mw:(r + 1) * mw].cpu().tolist()
                hidden = [c for c in range(lay["q"]) if not (words[c // 32] >> (c % 32)) & 1]
                if hidden:
                    c = hidden[0]
                    v = (words[c // 32] ^ (1 << (c % 32))) & 0xFFFFFFFF
                    eng.rowmask[r * mw + c // 32] = v - (1 << 32) if v >= 1 << 31 else v
            elif fault == "pos":
                eng.pos[last_level0] += 1
            elif fault == "lm_swap" and lay["tiny"] >= 2:
                eng.lm_rows[[1, 2]] = eng.lm_rows[[2, 1]]
        return rope(stream, l, *a)

    def commit(stream, commit_):
        assert commit_ is True and eng.DW == 1
        lay = _layout_now(eng)
        check(eng.lib.lade_accept_update(eng._ctx, stream, _ptr(eng.am), _ptr(eng.meta), _ptr(eng.res)), "accept")
        n_layers = eng.L
        if fault == "kv_shift":
            res = eng.res.cpu().tolist()
            mh, src = res[_cabi.R_MAX_HIT], res[_cabi.R_KV_SRC]
            if mh > 0 and src + mh + 1 <= lay["kv"] + lay["q"]:              # reads only rows written this step
                eng.res[_cabi.R_KV_SRC] += 1
        elif fault == "kv_layers":
            n_layers = eng.L - 1
        check(eng.lib.lade_kv_compact(stream, _ptr(eng.res), _ptr(eng.kv[0, 0]), _ptr(eng.kv[0, 1]), eng.kv.stride(0),
                                      n_layers, eng.nkv, eng.kv_capacity, eng.D, max(eng.GS - 1, 1)), "compact")
        return 2

    if fault in ("mask", "pos", "lm_swap"):
        eng._rope_append = rope_after_layout
    elif fault in ("kv_shift", "kv_layers"):
        eng._commit = commit
    elif fault == "qk_norm":
        eng.q_norm_w = [eng.q_norm_w[0]] * eng.L
        eng.k_norm_w = [eng.k_norm_w[0]] * eng.L
    return eng


# A window row's position off by one is planted on Qwen3: on the random-init Llama attention is nearly uniform, so the
# shift moves that row's logits by only 2.2 / 2.5 (rms / max ratio, measured on an H100), inside R; Qwen3's q/k norms
# give scores of several units, where one position moves the row far.
#            fault        case             the check that must fail
PLANTS = [("mask", "llama_mha", "logits"),
          ("pos", "qwen3_impl3", "logits"),
          ("lm_swap", "llama_mha", "logits"),
          ("kv_shift", "periodic_bf16", "kv"),
          ("kv_layers", "periodic_bf16", "kv"),
          ("qk_norm", "qwen3_impl3", "logits")]


@pytest.mark.parametrize("fault,name,check_kind", PLANTS, ids=[p[0] for p in PLANTS])
def test_planted_fault_fails_the_checks(fault, name, check_kind):
    eng = plant(make_engine(name, use_cuda_graph=False), fault)
    rep = run_lockstep(name, [eng])
    honest = HONEST.get(name)
    print(f"\nplanted {fault} on {rep.line()}" +
          (f"; honest worst logits {honest.logit_rms:.2f}/{honest.logit_max:.2f} KV {honest.kv_rms:.2f}/"
           f"{honest.kv_max:.2f}" if honest else ""))
    for f in rep.failures[:6]:
        print("   ", f)
    assert check_kind in rep.kinds(), rep.line()
    eng.close()


@pytest.mark.parametrize("fault,name", [p[:2] for p in PLANTS[:3]], ids=[p[0] for p in PLANTS[:3]])
def test_planted_fault_keeps_ids_within_the_tie_allowance(fault, name):
    """The id comparison the other engine tests use does not see these faults."""
    from test_gpu_e2e import assert_same_or_tie
    _, ocfg, w = build(name)
    _, _, _, W, N, G, P, new, _, _ = CASES[name]
    prompt = prompt_of(name)
    honest = make_engine(name, use_cuda_graph=False)
    want = honest.generate(prompt, new, rng=random.Random(5))
    eng = plant(make_engine(name, use_cuda_graph=False, pipeline_host=False), fault)
    got = eng.generate(prompt, new, rng=random.Random(5))
    div = assert_same_or_tie(got, want, ocfg, w, f"planted {fault}")
    print(f"\nplanted {fault}: ids {'identical' if div is None else f'diverge at {div} on a tie'}; steps "
          f"{eng.last_steps} (honest {honest.last_steps})")
    honest.close()
    eng.close()
