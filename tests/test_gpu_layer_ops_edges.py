"""The decoder layer's glue kernels at their edges, bf16 and (through the _f16 entry points) fp16.

* lade_rmsnorm / lade_rmsnorm_gather against oracle.llama_ref.rms_norm_fp64: every element is the float64 value rounded,
  or its stated alternative; hidden from 8 through the strided loops (> 8192) and the shared-memory opt-in (> 12288) to
  the 24576 limit; zero rows, one huge element, fp16 rows at +-60000, rows of 1e-4; in place as the engine calls it;
* lade_rope_append bit for bit at 1536 work items per row (the loop path), clamped positions, and a step that crosses
  kv_capacity: the rows that fit land, the rest are dropped, Q is complete, canaries around everything;
* lade_swiglu against swiglu_fp64 through the grid-stride loop, with gates at +-120, +-88.5, +-0, subnormals and an
  overflowing fp16 product;
* lade_argmax_rows against a lowest-index argmax in float64: -inf holes, an all -inf row, +inf twice, the maximum in
  the scalar tail, padding columns holding the dtype's maximum, vocab 1 .. 128256;
* lade_kv_compact on 16-bit patterns with a padded layer stride, max_rows around the hit count, src < 0, no hit, and
  ranges that end on the last cache row: every other byte unchanged; and its precondition (source and destination rows
  do not overlap) on every step of the reference traces."""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import llama_ref as LR
from test_dense_bound import DTYPES, norm_data, swiglu_data

pytestmark = pytest.mark.gpu
CANARY = 777.0
EPS = 1e-5


def _lib():
    from lookaheaddecoding_b200 import _cabi
    return _cabi.load(), _cabi


def _fn(name, dtype):
    lib, _ = _lib()
    return getattr(lib, name if dtype == torch.bfloat16 else name + "_f16")


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _gen(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


def _guarded(rows, cols, dtype):
    """[rows + 1, cols] of CANARY; kernels write the first `rows` rows."""
    return torch.full((rows + 1, cols), CANARY, dtype=dtype, device="cuda")


def _is_canary(t):
    return bool((t == CANARY).all())


# ---- RMSNorm --------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtn", list(DTYPES))
@pytest.mark.parametrize("hidden", [8, 264, 4096, 5120, 8192, 12288, 16384, 24576])
def test_rmsnorm_has_no_unexplained_element(hidden, dtn):
    _, cabi = _lib()
    dtype = DTYPES[dtn]
    fn = _fn("lade_rmsnorm", dtype)
    took = total = 0
    for rows in (1, 128, 257):
        x, d, w = norm_data(rows, hidden, dtype, _gen(hidden + rows), "cuda")
        x0, d0 = x.clone(), d.clone()
        # plain
        out = _guarded(rows, hidden, dtype)
        cabi.check(fn(_stream(), x.data_ptr(), 0, w.data_ptr(), 0, out.data_ptr(), rows, hidden, EPS))
        torch.cuda.synchronize()
        _, ref, alt = LR.rms_norm_fp64(x, None, w, EPS, dtype)
        bad, used = LR.unexplained(out[:rows], ref, alt)
        assert bad == 0, f"hidden {hidden} rows {rows}: {bad} elements are neither rounding of the float64 value"
        assert torch.equal(x, x0) and _is_canary(out[rows:])
        took, total = took + used, total + ref.numel()
        # residual add, h written over x as the engine does
        h_ref, ref, alt = LR.rms_norm_fp64(x0, d, w, EPS, dtype)
        out = _guarded(rows, hidden, dtype)
        h = _guarded(rows, hidden, dtype)
        h[:rows] = x0
        cabi.check(fn(_stream(), h.data_ptr(), d.data_ptr(), w.data_ptr(), h.data_ptr(), out.data_ptr(), rows, hidden, EPS))
        torch.cuda.synchronize()
        assert torch.equal(h[:rows], h_ref), "h_out is not T(x + delta)"
        bad, used = LR.unexplained(out[:rows], ref, alt)
        assert bad == 0, f"hidden {hidden} rows {rows} with delta: {bad} unexplained elements"
        assert torch.equal(d, d0) and _is_canary(out[rows:]) and _is_canary(h[rows:])
        took, total = took + used, total + ref.numel()
    print(f"rmsnorm {dtn} hidden {hidden}: {took} of {total} elements took the rounding alternative")


@pytest.mark.parametrize("dtn", list(DTYPES))
@pytest.mark.parametrize("hidden", [264, 4096, 16384])
def test_rmsnorm_gather_against_the_float64_reference(hidden, dtn):
    _, cabi = _lib()
    dtype = DTYPES[dtn]
    fn = _fn("lade_rmsnorm_gather", dtype)
    rows = 128
    x, d, w = norm_data(rows, hidden, dtype, _gen(hidden), "cuda")
    x0, d0 = x.clone(), d.clone()
    idx = torch.tensor([127, 0, 5, 5, 127, 64, 3, 2, 1, 0, 126, 127], dtype=torch.int32, device="cuda")
    for delta in (None, d):
        out = _guarded(idx.numel(), hidden, dtype)
        cabi.check(fn(_stream(), x.data_ptr(), 0 if delta is None else delta.data_ptr(), w.data_ptr(), idx.data_ptr(),
                      out.data_ptr(), idx.numel(), hidden, EPS))
        torch.cuda.synchronize()
        _, ref, alt = LR.rms_norm_fp64(x0[idx.long()], None if delta is None else d0[idx.long()], w, EPS, dtype)
        bad, used = LR.unexplained(out[:idx.numel()], ref, alt)
        print(f"rmsnorm_gather {dtn} hidden {hidden} delta {delta is not None}: {used} of {ref.numel()} took the alternative")
        assert bad == 0
        assert torch.equal(x, x0) and torch.equal(d, d0) and _is_canary(out[idx.numel():])
        assert torch.equal(out[2], out[3]) and torch.equal(out[0], out[4])


@pytest.mark.parametrize("dtn", list(DTYPES))
def test_rmsnorm_shape_errors(dtn):
    _, cabi = _lib()
    dtype = DTYPES[dtn]
    x = torch.zeros(2, 24584, dtype=dtype, device="cuda")
    out = _guarded(2, 24584, dtype)
    idx = torch.zeros(2, dtype=torch.int32, device="cuda")
    for hidden, code in [(24584, cabi.LADE_EUNSUPPORTED), (12, cabi.LADE_EINVAL), (0, cabi.LADE_EINVAL)]:
        assert _fn("lade_rmsnorm", dtype)(_stream(), x.data_ptr(), 0, x.data_ptr(), 0, out.data_ptr(), 2, hidden, EPS) == code
        assert _fn("lade_rmsnorm_gather", dtype)(_stream(), x.data_ptr(), 0, x.data_ptr(), idx.data_ptr(), out.data_ptr(), 2,
                                                 hidden, EPS) == code
    torch.cuda.synchronize()
    assert _is_canary(out)


# ---- RoPE + append --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtn", list(DTYPES))
@pytest.mark.parametrize("over", [0, 5])
@pytest.mark.parametrize("nh,nkv,D", [(64, 64, 128), (64, 8, 128), (32, 8, 64)])
def test_rope_append_clamps_positions_and_drops_rows_past_the_capacity(nh, nkv, D, over, dtn):
    """`over` rows of the step do not fit the cache: they are dropped, not written past the head's slab."""
    _, cabi = _lib()
    dtype = DTYPES[dtn]
    rows, q_pad, max_pos, kv_len = 37, 40, 512, 61
    cap = kv_len + rows - over
    gen = _gen(nh + D + over)
    qkv = torch.randn(rows, (nh + 2 * nkv) * D, generator=gen, device="cuda").to(dtype)
    cos, sin = LR.rope_tables(D, max_pos, 10000.0, dtype, "cuda")
    pos = torch.randint(0, max_pos, (rows,), generator=gen, device="cuda").to(torch.int32)
    qkv[1] = qkv[0]
    qkv[3] = qkv[4] = qkv[2]
    pos[:6] = torch.tensor([-3, 0, max_pos - 1, max_pos, max_pos + 7, -2 ** 31], dtype=torch.int32, device="cuda")
    meta = torch.zeros(cabi.META_INTS, dtype=torch.int32, device="cuda")
    meta[cabi.M_KV_LEN] = kv_len
    qo = torch.full((nh, q_pad, D), CANARY, dtype=dtype, device="cuda")
    # one flat buffer per cache, 8 canary rows behind the last head's slab
    kbuf = torch.full(((nkv * cap + 8) * D,), CANARY, dtype=dtype, device="cuda")
    vbuf = torch.full(((nkv * cap + 8) * D,), CANARY, dtype=dtype, device="cuda")
    cabi.check(_fn("lade_rope_append", dtype)(_stream(), qkv.data_ptr(), cos.data_ptr(), sin.data_ptr(), pos.data_ptr(),
                                              meta.data_ptr(), qo.data_ptr(), kbuf.data_ptr(), vbuf.data_ptr(), rows, q_pad,
                                              nh, nkv, D, cap, max_pos))
    torch.cuda.synchronize()
    q = qkv[:, : nh * D].view(rows, nh, D).transpose(0, 1)
    k = qkv[:, nh * D:(nh + nkv) * D].view(rows, nkv, D).transpose(0, 1)
    v = qkv[:, (nh + nkv) * D:].view(rows, nkv, D).transpose(0, 1)
    p = pos.long().clamp(0, max_pos - 1)
    c, s = cos[p], sin[p]
    q_ref = (q * c) + (LR.rotate_half(q) * s)            # modeling_llama.py:344-345, every op in the model dtype
    k_ref = (k * c) + (LR.rotate_half(k) * s)
    assert torch.equal(qo[:, :rows], q_ref), "Q is incomplete or wrong"
    kc = kbuf[: nkv * cap * D].view(nkv, cap, D)
    vc = vbuf[: nkv * cap * D].view(nkv, cap, D)
    # rows 0 / 1 and rows 2 / 3 / 4 carry the same data: a clamped position gives the row of position 0 / max_pos - 1
    assert torch.equal(qo[:, 0], qo[:, 1]) and torch.equal(qo[:, 2], qo[:, 3]) and torch.equal(qo[:, 2], qo[:, 4])
    assert torch.equal(kc[:, kv_len], kc[:, kv_len + 1]) and torch.equal(kc[:, kv_len + 2], kc[:, kv_len + 4])
    assert _is_canary(qo[:, rows:]), "pad rows of q_out were written"
    fit = rows - over
    assert torch.equal(kc[:, kv_len:], k_ref[:, :fit]) and torch.equal(vc[:, kv_len:], v[:, :fit])
    assert _is_canary(kc[:, :kv_len]) and _is_canary(vc[:, :kv_len]), "a dropped row landed in the next head's slab"
    assert _is_canary(kbuf[nkv * cap * D:]) and _is_canary(vbuf[nkv * cap * D:]), "a dropped row landed past the cache"


# ---- SwiGLU ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtn", list(DTYPES))
@pytest.mark.parametrize("rows,inter", [(53, 11008), (128, 27648), (1, 8), (3, 1376)])
def test_swiglu_has_no_unexplained_element(rows, inter, dtn):
    _, cabi = _lib()
    dtype = DTYPES[dtn]
    gu = swiglu_data(rows, inter, dtype, _gen(inter), "cuda")
    gu0 = gu.clone()
    out = _guarded(rows, inter, dtype)
    cabi.check(_fn("lade_swiglu", dtype)(_stream(), gu.data_ptr(), out.data_ptr(), rows, inter))
    torch.cuda.synchronize()
    ref, alt = LR.swiglu_fp64(gu, dtype)
    bad, used = LR.unexplained(out[:rows], ref, alt)
    print(f"swiglu {dtn} [{rows}, {inter}]: {used} of {ref.numel()} elements took the rounding alternative")
    assert bad == 0, f"{bad} elements are neither rounding of the float64 value"
    assert not torch.isnan(ref.float()).any() and not torch.isnan(out[:rows].float()).any()
    assert torch.equal(gu, gu0) and _is_canary(out[rows:])
    if dtype == torch.float16 and inter >= 16:
        assert torch.isinf(out[0, 13]) and torch.isinf(ref[0, 13])


# ---- argmax ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtn", list(DTYPES))
@pytest.mark.parametrize("vocab", [1, 7, 8, 1000, 32000, 128256])
def test_argmax_rows_with_infinities_tails_and_padding(vocab, dtn):
    _, cabi = _lib()
    dtype = DTYPES[dtn]
    inf = float("inf")
    rows = 9
    for ld in (vocab, vocab + 3, vocab + 8):
        x = (torch.randn(rows, ld, generator=_gen(vocab + ld), device="cuda") * 4).round()
        x[1, ::3] = -inf
        x[2] = -inf
        if vocab >= 3:
            x[3, vocab // 2] = x[3, vocab - 2] = inf
        x[4, vocab - 1] = 100.0
        x[5, 0] = x[5, vocab - 1] = 100.0
        x[6] = -inf
        x[6, vocab - 1] = -1000.0
        x[7, : vocab - 1] = -inf                       # the only finite entry is the last one
        x[8, 0] = -0.0
        x[:, vocab:] = torch.finfo(dtype).max          # padding columns must not compete
        x = x.to(dtype)
        out = torch.full((rows + 1,), -5, dtype=torch.int32, device="cuda")
        cabi.check(_fn("lade_argmax_rows", dtype)(_stream(), x.data_ptr(), rows, vocab, ld, out.data_ptr()))
        xd = x[:, :vocab].double().cpu()
        at_max = xd == xd.max(-1, keepdim=True).values
        want = torch.where(at_max, torch.arange(vocab), vocab).min(-1).values
        assert out[:rows].cpu().tolist() == want.tolist(), f"vocab {vocab} ld {ld}"
        assert out[rows].item() == -5
        assert want[2] == 0 and want[5] == 0 and want[6] == vocab - 1


# ---- KV compaction --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("D", [64, 128])
def test_kv_compact_moves_exactly_the_hit_rows(D):
    """Payloads are random 16-bit patterns (the kernel moves bits, so they stand for bf16 and fp16 alike)."""
    lib, cabi = _lib()
    L, nkv, cap, pad = 3, 2, 64, 64
    slab = nkv * cap * D
    stride = 2 * slab + pad
    gen = _gen(D)
    cases = [  # (max_hit, src, dst, max_rows)
        (3, 40, 11, 1), (3, 40, 11, 2), (3, 40, 11, 3), (3, 40, 11, 5),
        (3, -1, 11, 3), (0, 40, 11, 3), (4, cap - 4, 20, 4), (4, 10, cap - 4, 4), (1, 12, 11, 1), (3, 40, 11, 0),
    ]
    for max_hit, src, dst, max_rows in cases:
        buf = torch.randint(-32768, 32768, (L, stride), generator=gen, device="cuda").to(torch.int16)
        want = buf.clone()
        moved = min(max_hit, max_rows) if src >= 0 else 0
        live, live_want = (t[:, : 2 * slab].view(L, 2, nkv, cap, D) for t in (buf, want))
        if moved > 0:
            live_want[:, :, :, dst:dst + moved] = live[:, :, :, src:src + moved]
        res = torch.zeros(cabi.RES_INTS, dtype=torch.int32, device="cuda")
        res[cabi.R_MAX_HIT], res[cabi.R_KV_SRC], res[cabi.R_KV_DST] = max_hit, src, dst
        cabi.check(lib.lade_kv_compact(_stream(), res.data_ptr(), buf.data_ptr(), buf.data_ptr() + 2 * slab, stride, L, nkv,
                                       cap, D, max_rows))
        torch.cuda.synchronize()
        assert torch.equal(buf, want), f"hit {max_hit} src {src} dst {dst} max_rows {max_rows}"


def test_accepted_rows_never_overlap_their_destination():
    """lade_kv_compact copies every row in its own CTA, which is only right when [src, src + hit) and [dst, dst + hit)
    do not overlap: on every step of the reference traces, R_KV_SRC - R_KV_DST >= R_MAX_HIT."""
    from helpers import make_lade_config
    from test_gpu_state_machine import CASES
    lib, cabi = _lib()
    checked = 0
    i32 = dict(dtype=torch.int32, device="cuda")
    for name, c in sorted(CASES.items()):
        W, N, G = c["W"], c["N"], c["G"]
        GS, WCAP = N - 1, W + N - 3
        P = len(c["prompt"])
        max_length = P + c["max_new"]
        eos = [c["eos_token_id"]] if c["eos_token_id"] is not None else []
        cfg = make_lade_config(W, N, G, c["model"]["vocab"], max_length + N + 8, pool=c["pool_from_prompt"], eos=eos)
        ctx = C.c_void_p()
        cabi.check(lib.lade_ctx_create(C.byref(cfg), C.byref(ctx)), "create")
        prompt = np.asarray(c["prompt"], dtype=np.int32)
        win0 = np.asarray(c["steps"][0]["past_tokens"][0], dtype=np.int32)
        cabi.check(lib.lade_ctx_reset(ctx, _stream(), prompt.ctypes.data, P, win0.ctypes.data, WCAP, max_length), "reset")
        lm_cap = 1 + WCAP + G * GS
        q_pad = max(P + WCAP, GS * (W + G)) + 8
        mw = (q_pad + 31) // 32 + 1
        ids, pos, rd = torch.zeros(q_pad, **i32), torch.zeros(q_pad, **i32), torch.zeros(q_pad, **i32)
        lm_rows, meta = torch.zeros(lm_cap, **i32), torch.zeros(cabi.META_INTS, **i32)
        rowmask, res = torch.zeros(q_pad * mw, **i32), torch.zeros(cabi.RES_INTS, **i32)
        for i, g in enumerate(c["steps"]):
            cabi.check(lib.lade_step_layout(ctx, _stream(), q_pad, ids.data_ptr(), pos.data_ptr(), rd.data_ptr(),
                                            lm_rows.data_ptr(), meta.data_ptr(), rowmask.data_ptr(), mw), "layout")
            am = np.zeros(lm_cap, dtype=np.int32)
            am[0] = g["first_guess"]
            am[1:1 + len(g["inp_tokens"])] = g["inp_tokens"]
            am[1 + WCAP:1 + WCAP + len(g["guess_results"])] = g["guess_results"]
            am_d = torch.from_numpy(am).cuda()
            cabi.check(lib.lade_accept_update(ctx, _stream(), am_d.data_ptr(), meta.data_ptr(), res.data_ptr()), "accept")
            r = res.cpu().numpy()
            hit, src, dst = int(r[cabi.R_MAX_HIT]), int(r[cabi.R_KV_SRC]), int(r[cabi.R_KV_DST])
            if hit > 0 and src >= 0:
                assert src - dst >= hit, f"{name} step {i}: src {src} dst {dst} hit {hit}"
                checked += 1
        assert r[cabi.R_DONE], name
        lib.lade_ctx_destroy(ctx)
    print(f"kv_compact precondition held on {checked} steps with a hit")
    assert checked > 0
