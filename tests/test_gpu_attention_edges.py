"""lade_attn_fwd at its edges, launched the way the engine launches it.

* exact mask probes: Q = 0 makes every visible probability equal, one-hot V columns read the mask back bit by bit;
* one CUDA graph replayed while meta[KV_LEN] walks through word, tile and split boundaries (the kernel derives its tile
  partition, the zeroing of stale V rows and its prefetch from that value at run time);
* peaked scores from integer Q and K (exact dot products): an attention sink, a row maximum that appears in the last
  tile of the last split, the maximum inside the step block, a split whose merge weight underflows to 0;
* shape edges: T == kv_capacity, PAD rows inside q_pad, GQA 8:1, 40 heads, more splits than KV tiles, guard rows after
  the output;
* programmatic-dependent-launch chains captured in one graph (rope_append -> attention, 32 attentions on one scratch)
  must write the same bits as the same launches serialised.
Values are checked against oracle.llama_ref.attention_fp64 and its per-element bound; PAD rows (q_len <= row < q_pad)
see the cache and nothing of the step, as the engine's row mask has them."""
import numpy as np
import pytest
import torch

from oracle import llama_ref as LR
from oracle import lookahead as LA

pytestmark = pytest.mark.gpu
DTYPES = {"bf16": torch.bfloat16, "fp16": torch.float16}
IMPLS = [1, 2, 3]
SENTINEL = 12345.0
GUARD = 4


def _lib():
    from lookaheaddecoding_b200 import _cabi
    return _cabi, _cabi.load()


def _steady(W=15, N=5, g=15):
    gs = N - 1
    return LA.layout_from_shape([W - 1] + [W] * (N - 2), 1, g * gs, gs)


def _impl3_fits(T, splits):
    return T <= 384 * min(splits, 8)


class Launch:
    """Fixed buffers of one lade_attn_fwd call site (what a captured graph points at)."""

    def __init__(self, lay, q_pad, Hq, Hkv, cap, splits, impl, dt, D=128):
        c, self.lib = _lib()
        self.c, self.lay, self.q_pad, self.Hq, self.Hkv, self.cap = c, lay, q_pad, Hq, Hkv, cap
        self.splits, self.impl, self.dt, self.D = splits, impl, dt, D
        self.q = torch.zeros(Hq, q_pad, D, dtype=dt, device="cuda")
        self.k = torch.full((Hkv, cap, D), float("nan"), dtype=dt, device="cuda")
        self.v = torch.full((Hkv, cap, D), float("nan"), dtype=dt, device="cuda")
        self.out_full = torch.full((q_pad + GUARD, Hq * D), SENTINEL, dtype=dt, device="cuda")
        self.out = self.out_full[:q_pad]
        self.meta = torch.zeros(c.META_INTS, dtype=torch.int32, device="cuda")
        self.mw = (q_pad + 31) // 32 + 1
        bits = np.zeros((q_pad, self.mw * 32), dtype=bool)
        bits[:lay.q_len, :lay.q_len] = LA.step_mask(lay)         # PAD rows: all zero, as lade_step_layout writes them
        words = np.packbits(bits.reshape(q_pad, self.mw, 32), axis=-1, bitorder="little").view(np.uint32)
        self.rowmask = torch.from_numpy(words.reshape(q_pad, self.mw).view(np.int32).copy()).cuda()
        self.scratch = torch.zeros(self.lib.lade_attn_scratch_bytes(q_pad, Hq, D, splits), dtype=torch.uint8, device="cuda")

    def set_meta(self, kv_len):
        c, lay = self.c, self.lay
        vals = {c.M_Q_LEN: lay.q_len, c.M_KV_LEN: kv_len, c.M_N_INPUT: lay.n_input, c.M_LEVEL_OFFSET: lay.level_offset,
                c.M_ALL_OFFSET: lay.level_offset + lay.dist_offset, c.M_TINY: lay.tiny, c.M_N_LEVELS: len(lay.level_sizes),
                c.M_N_GUESS_TOK: lay.n_guess_tok, c.M_IS_PREFILL: 0, c.M_Q_PAD: self.q_pad, c.M_PHASE: 2}
        m = torch.zeros(c.META_INTS, dtype=torch.int32)
        for key, val in vals.items():
            m[key] = val
        self.meta.copy_(m)

    def launch(self, kv_bound):
        fwd = self.lib.lade_attn_fwd if self.dt == torch.bfloat16 else self.lib.lade_attn_fwd_f16
        self.c.check(fwd(torch.cuda.current_stream().cuda_stream, self.q.data_ptr(), self.k.data_ptr(), self.v.data_ptr(),
                         self.out.data_ptr(), self.rowmask.data_ptr(), self.mw, self.meta.data_ptr(),
                         self.scratch.data_ptr(), self.q_pad, self.Hq, self.Hkv, self.D, self.cap, kv_bound, self.splits,
                         self.impl), "lade_attn_fwd")

    def fill(self, kv_len, gen, peaked=None):
        """This step's Q (every q_pad row) and K/V rows [0, T) random, the rows past T NaN (stale cache)."""
        T = kv_len + self.lay.q_len
        self.q.copy_(torch.randn(self.Hq, self.q_pad, self.D, generator=gen).to(self.dt))
        self.k.fill_(float("nan"))
        self.v.fill_(float("nan"))
        self.k[:, :T] = torch.randn(self.Hkv, T, self.D, generator=gen).to(self.dt).cuda()
        self.v[:, :T] = torch.randn(self.Hkv, T, self.D, generator=gen).to(self.dt).cuda()

    def check(self, kv_len, what):
        """The rows [0, q_pad) against the float64 reference, the guard rows untouched, the split counters back at 0."""
        T = kv_len + self.lay.q_len
        torch.cuda.synchronize()
        assert torch.all(self.out_full[self.q_pad:] == SENTINEL), f"{what}: write past out[q_pad]"
        assert int(self.scratch[:65536].view(torch.int32).abs().sum()) == 0, f"{what}: split counters must self-reset"
        vis = LR.visibility(torch.from_numpy(LA.step_mask(self.lay)), kv_len, self.q_pad).cuda()
        o_ref, bound = LR.attention_fp64(self.q, self.k[:, :T], self.v[:, :T], vis, self.dt)
        got = self.out.view(self.q_pad, self.Hq, self.D).transpose(0, 1)
        ok, mx, mean = LR.within_bound(got, o_ref, bound)
        assert ok, f"{what}: err/bound max {mx:.3f} mean {mean:.3f}"
        return mx


def _report(name, worst):
    print(f"\n{name}: worst err/bound {worst:.3f}")


# ---- 1. exact mask probes -------------------------------------------------------------------------------------------
PROBE_KV = [0, 5, 31, 100, 127, 130, 250, 383, 1278, 3001]


@pytest.mark.parametrize("dtn", list(DTYPES))
@pytest.mark.parametrize("impl", IMPLS)
def test_mask_probes_are_exact(impl, dtn):
    """Q = 0: every visible score is 0, every visible p is 1 / (visible count).  Probe column i (all step columns and the
    cache columns just below kv_len) has V = e_i, so o[row, i] is exactly T(1 / count) if the row sees it and exactly 0
    if it does not -- no tolerance.  The stale rows past T are NaN, so a column wrongly seen past T shows up too."""
    dt = DTYPES[dtn]
    lay = _steady(g=12)                                   # 108 step rows, 8 PAD rows
    q_len, q_pad, Hq, Hkv = lay.q_len, lay.q_len + 8, 4, 2
    for kv_len in PROBE_KV:
        T = kv_len + q_len
        splits = 4 if impl != 3 else max(4, -(-T // 384))
        if impl == 3 and not _impl3_fits(T, splits):
            continue
        L = Launch(lay, q_pad, Hq, Hkv, T + 40, splits, impl, dt)
        L.set_meta(kv_len)
        n_cache = min(kv_len, 128 - q_len)
        probes = list(range(kv_len - n_cache, T))
        L.k[:, :T] = torch.randn(Hkv, T, 128).to(dt).cuda()
        L.v[:, :T] = 0
        for i, col in enumerate(probes):
            L.v[:, col, i] = 1
        L.launch(T)
        torch.cuda.synchronize()
        assert torch.all(L.out_full[q_pad:] == SENTINEL)
        vis = LR.visibility(torch.from_numpy(LA.step_mask(lay)), kv_len, q_pad)
        count = vis.sum(-1).double()
        want = torch.zeros(q_pad, 128, dtype=torch.float64)
        want[:, :len(probes)] = torch.where(vis[:, probes], (1.0 / count.clamp_min(1)).unsqueeze(-1), 0.0)
        want = want.to(dt)
        got = L.out.view(q_pad, Hq, 128).cpu()
        for h in range(Hq):
            bad = (got[:, h] != want).nonzero()
            assert bad.numel() == 0, f"kv {kv_len} head {h}: {bad.shape[0]} wrong, first (row, probe) {bad[0].tolist()}"


# ---- 2. one captured launch, kv_len swept under it ------------------------------------------------------------------
SWEEP_KV = [0, 1, 2, 127, 128, 129, 255, 256, 257, 383, 384, 385, 511, 512, 1023, 1024, 1025, 1278, 2047, 2048,
            3071, 3072, 3073]


@pytest.mark.parametrize("splits", [1, 3, 4, 8])
@pytest.mark.parametrize("dtn", list(DTYPES))
@pytest.mark.parametrize("impl", IMPLS)
def test_kv_sweep_under_one_graph(impl, dtn, splits):
    dt = DTYPES[dtn]
    lay = _steady()
    q_len, q_pad = lay.q_len, lay.q_len + 8
    kvs = [kv for kv in SWEEP_KV if impl != 3 or _impl3_fits(kv + q_len, splits)]
    if not kvs:
        pytest.skip("impl 3 holds no kv_len of the sweep with one split")
    T_max = max(kvs) + q_len
    L = Launch(lay, q_pad, 4, 2, T_max + 70, splits, impl, dt)
    gen = torch.Generator().manual_seed(splits * 10 + impl)
    L.set_meta(kvs[0])
    L.fill(kvs[0], gen)
    L.launch(T_max)                                       # warm-up (kernel attributes, tensor maps) outside the capture
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        L.launch(T_max)
    worst = 0.0
    for kv_len in kvs:
        L.set_meta(kv_len)
        L.fill(kv_len, gen)
        graph.replay()
        worst = max(worst, L.check(kv_len, f"impl {impl} {dtn} splits {splits} kv {kv_len}"))
    _report(f"sweep impl {impl} {dtn} splits {splits}", worst)


# ---- 3. peaked scores from exact integer inputs ---------------------------------------------------------------------
def _peaked_inputs(case, kv_len, lay, Hq, Hkv, splits, dt, gen):
    """Integer Q and K: every fp32 partial sum of Q.K is an exact integer, so T(raw) does not depend on summation order.
    Dimensions 32.. hold random {-1, 0, 1}; dimensions 0..31 carry a level: q = 2 there, a column of level L has k = L,
    adding 64 L to its raw score (L = 4: scaled score about +22.6, L = -18: about -102)."""
    T = kv_len + lay.q_len
    q = torch.randint(-1, 2, (Hq, lay.q_len + 8, 128), generator=gen).float()
    k = torch.randint(-1, 2, (Hkv, T, 128), generator=gen).float()
    q[:, :, :32] = 2
    k[:, :, :32] = 0
    level = torch.zeros(T)
    level[torch.randperm(T, generator=gen)[: T // 8]] = -4          # a spread of low scores in every case
    if case == "sink":
        level[0] = 4
    elif case == "late_max":                                         # the input token's column, in the last tile
        level[kv_len] = 4
    elif case == "step_max":                                         # a window column only some rows see
        level[kv_len + 1 + lay.level_sizes[0] + 2] = 4
    elif case == "dead_split":                                       # every column of split 0 about 100 below
        n_tiles = -(-T // 128)
        base, rem = divmod(n_tiles, splits)
        level[: 128 * (base + (rem > 0))] = -18
    k[:, :, :32] = level.view(1, T, 1)
    v = torch.randn(Hkv, T, 128, generator=gen)
    return q.to(dt), k.to(dt), v.to(dt)


@pytest.mark.parametrize("case", ["sink", "late_max", "step_max", "dead_split"])
@pytest.mark.parametrize("dtn", list(DTYPES))
@pytest.mark.parametrize("impl", IMPLS)
def test_peaked_scores(impl, dtn, case):
    dt = DTYPES[dtn]
    lay = _steady()
    kv_len, splits, Hq, Hkv = 1280, 4, 4, 2           # 11 tiles: splits of 3, 3, 3, 2; the last tile holds the step block
    T = kv_len + lay.q_len
    q_pad = lay.q_len + 8
    L = Launch(lay, q_pad, Hq, Hkv, T + 70, splits, impl, dt)
    q, k, v = _peaked_inputs(case, kv_len, lay, Hq, Hkv, splits, dt, torch.Generator().manual_seed(len(case)))
    L.q.copy_(q)
    L.k[:, :T], L.v[:, :T] = k.cuda(), v.cuda()
    L.set_meta(kv_len)
    L.launch(T)
    _report(f"peaked {case} impl {impl} {dtn}", L.check(kv_len, f"peaked {case} impl {impl} {dtn}"))


# ---- 4. shape edges -------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtn", list(DTYPES))
@pytest.mark.parametrize("impl", IMPLS)
def test_cache_full_to_capacity(impl, dtn):
    """T == kv_capacity: the last tile reads past the tensor (the TMA fills those rows with zeros)."""
    dt = DTYPES[dtn]
    lay = _steady()
    worst = 0.0
    for kv_len in (392, 400, 1160, 1170):                # T = 512, 520, 1280, 1290
        T = kv_len + lay.q_len
        L = Launch(lay, lay.q_len, 4, 2, T, 4, impl, dt)
        L.set_meta(kv_len)
        L.fill(kv_len, torch.Generator().manual_seed(kv_len))
        L.launch(T)
        worst = max(worst, L.check(kv_len, f"T == capacity {T} impl {impl} {dtn}"))
    _report(f"T == capacity impl {impl} {dtn}", worst)


# (W, N, guesses g < G) -> q_len; q_pad adds PAD rows up to the row count of the fixed-shape step
PAD_SHAPES = [((5, 3, 1), 16), ((10, 4, 2), 64), ((10, 4, 2), 65), ((15, 5, 5), 120), ((15, 5, 5), 128),
              ((15, 5, 5), 129), ((20, 7, 10), 240)]


@pytest.mark.parametrize("dtn", list(DTYPES))
@pytest.mark.parametrize("impl", IMPLS)
def test_pad_rows_inside_q_pad(impl, dtn):
    dt = DTYPES[dtn]
    worst = 0.0
    for (W, N, g), q_pad in PAD_SHAPES:
        lay = _steady(W, N, g)
        assert lay.q_len < q_pad
        for kv_len in (0, 300):
            T = kv_len + lay.q_len
            L = Launch(lay, q_pad, 4, 2, T + 70, 3, impl, dt)
            L.set_meta(kv_len)
            L.fill(kv_len, torch.Generator().manual_seed(q_pad + kv_len))
            L.launch(T)
            worst = max(worst, L.check(kv_len, f"q_pad {q_pad} kv {kv_len} impl {impl} {dtn}"))
    _report(f"PAD rows impl {impl} {dtn}", worst)


@pytest.mark.parametrize("dtn", list(DTYPES))
@pytest.mark.parametrize("impl", IMPLS)
@pytest.mark.parametrize("Hq,Hkv,kv_len,splits", [(8, 1, 700, 4), (40, 40, 517, 3), (40, 8, 1000, 3), (4, 2, 200, 8)])
def test_heads_and_splits(Hq, Hkv, kv_len, splits, impl, dtn):
    """GQA 8:1, 40 heads, and 8 splits over 3 KV tiles (5 splits have no tiles and must stay out of the merge)."""
    dt = DTYPES[dtn]
    lay = _steady()
    T = kv_len + lay.q_len
    if impl == 3 and not _impl3_fits(T, splits):
        pytest.skip("beyond impl 3's kv bound")
    L = Launch(lay, lay.q_len + 8, Hq, Hkv, T + 70, splits, impl, dt)
    L.set_meta(kv_len)
    L.fill(kv_len, torch.Generator().manual_seed(Hq * 100 + Hkv))
    L.launch(T)
    _report(f"Hq {Hq} Hkv {Hkv} splits {splits} impl {impl} {dtn}", L.check(kv_len, f"Hq {Hq} Hkv {Hkv} impl {impl}"))


@pytest.mark.parametrize("dtn", list(DTYPES))
def test_head_dim_64(dtn):
    """head_dim 64 runs on the mma.sync kernel (impl 0 picks it, impl 1 forces it)."""
    dt = DTYPES[dtn]
    lay = _steady()
    for impl in (0, 1):
        for kv_len in (0, 129, 1278):
            T = kv_len + lay.q_len
            L = Launch(lay, lay.q_len + 8, 4, 2, T + 70, 4, impl, dt, D=64)
            L.set_meta(kv_len)
            L.fill(kv_len, torch.Generator().manual_seed(kv_len + 64))
            L.launch(T)
            L.check(kv_len, f"head_dim 64 kv {kv_len} impl {impl} {dtn}")


# ---- 5. production launch chains under programmatic dependent launch -----------------------------------------------
def _with_pdl(enable, fn):
    _, lib = _lib()
    lib.lade_debug_attn_pdl(enable)
    try:
        return fn()
    finally:
        lib.lade_debug_attn_pdl(-1)


@pytest.mark.parametrize("dtn", list(DTYPES))
@pytest.mark.parametrize("impl", IMPLS)
def test_rope_append_then_attention_chain(impl, dtn):
    """lade_rope_append writes this step's Q and its K/V rows [kv_len, kv_len + q_pad); the attention that follows may
    start before it ends.  The new rows are NaN before the rope call, so any read that overtakes it shows up."""
    c, lib = _lib()
    dt = DTYPES[dtn]
    lay = _steady()
    kv_len, Hq, Hkv, D, max_pos = 1278, 4, 2, 128, 4096
    q_pad = lay.q_len + 8
    T = kv_len + lay.q_len
    L = Launch(lay, q_pad, Hq, Hkv, kv_len + q_pad + 70, 4, impl, dt)
    L.set_meta(kv_len)
    gen = torch.Generator().manual_seed(impl)
    L.fill(kv_len, gen)
    cache_k, cache_v = L.k[:, :kv_len].clone(), L.v[:, :kv_len].clone()
    qkv = torch.randn(q_pad, (Hq + 2 * Hkv) * D, generator=gen).to(dt).cuda()
    cos, sin = LR.rope_tables(D, max_pos, 10000.0, dt, "cuda")
    pos = torch.arange(kv_len, kv_len + q_pad, dtype=torch.int32, device="cuda")
    rope = lib.lade_rope_append if dt == torch.bfloat16 else lib.lade_rope_append_f16

    def reset():
        L.k.fill_(float("nan"))
        L.v.fill_(float("nan"))
        L.k[:, :kv_len], L.v[:, :kv_len] = cache_k, cache_v
        L.out_full.fill_(SENTINEL)

    def launches():
        s = torch.cuda.current_stream().cuda_stream
        c.check(rope(s, qkv.data_ptr(), cos.data_ptr(), sin.data_ptr(), pos.data_ptr(), L.meta.data_ptr(), L.q.data_ptr(),
                     L.k.data_ptr(), L.v.data_ptr(), q_pad, q_pad, Hq, Hkv, D, L.cap, max_pos), "lade_rope_append")
        L.launch(L.cap)

    def graphed():
        reset()
        launches()                                        # warm-up outside the capture
        torch.cuda.synchronize()
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            launches()
        reset()
        graph.replay()
        torch.cuda.synchronize()
        return L.out_full.clone()

    def serial():
        reset()
        launches()
        torch.cuda.synchronize()
        return L.out_full.clone()

    a = _with_pdl(1, graphed)
    b = _with_pdl(0, serial)
    assert torch.equal(a.view(torch.int16), b.view(torch.int16)), "PDL chain differs from the serialised launches"
    _report(f"rope -> attention impl {impl} {dtn}", L.check(kv_len, f"rope chain impl {impl} {dtn}"))


@pytest.mark.parametrize("dtn", list(DTYPES))
@pytest.mark.parametrize("impl", IMPLS)
def test_attention_chain_shares_one_scratch(impl, dtn):
    """32 back-to-back attention launches (one per layer), each with its own K/V and output, one scratch: a split merge
    of launch i + 1 must not see the partials of launch i."""
    dt = DTYPES[dtn]
    lay = _steady()
    kv_len, n = 700, 32
    T = kv_len + lay.q_len
    layers = []
    gen = torch.Generator().manual_seed(32 + impl)
    for i in range(n):
        L = Launch(lay, lay.q_len, 4, 2, T + 70, 4, impl, dt)
        L.set_meta(kv_len)
        L.fill(kv_len, gen)
        if i:
            L.scratch = layers[0].scratch
        layers.append(L)

    def launches():
        for L in layers:
            L.launch(T)

    def graphed():
        launches()
        torch.cuda.synchronize()
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            launches()
        for L in layers:
            L.out.zero_()
        graph.replay()
        torch.cuda.synchronize()
        return torch.stack([L.out_full.clone() for L in layers])

    def serial():
        for L in layers:
            L.out.zero_()
        launches()
        torch.cuda.synchronize()
        return torch.stack([L.out_full.clone() for L in layers])

    a = _with_pdl(1, graphed)
    b = _with_pdl(0, serial)
    assert torch.equal(a.view(torch.int16), b.view(torch.int16)), "PDL chain differs from the serialised launches"
    worst = max(L.check(kv_len, f"layer {i} impl {impl} {dtn}") for i, L in enumerate(layers))
    _report(f"32-launch chain impl {impl} {dtn}", worst)
