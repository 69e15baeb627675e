"""lade_rope_append_qknorm (Qwen3's per-head q/k RMSNorm fused into RoPE + KV append) against the float64 restatement of
tests/qknorm_restatement.py, in bf16 and fp16, at head_dim 128 and 64, with GQA and non-uniform norm weights that
differ between q and k:

* position 0 (cos 1, sin 0: the output is the norm itself): every element is the float64 value rounded, or its stated
  alternative;
* every position: every element is RoPE of one of the candidate combinations of its two inputs;
* more than 1024 work items per row (the loop path), rows of zeros, one huge element, fp16 rows near +-60000;
* clamped positions, a step that crosses kv_capacity with canaries around the caches, V bit-identical to the input,
  the unwritten rows of q_out keep their canaries;
* every argument error returns LADE_EINVAL and writes nothing.
"""
import pytest
import torch

import qknorm_restatement as Q
from oracle import llama_ref as LR

pytestmark = pytest.mark.gpu
DTYPES = {"bf16": torch.bfloat16, "fp16": torch.float16}
CANARY = 777.0
EPS = 1e-6
SHAPES = [(8, 2, 128), (8, 4, 64)]                     # (q heads, kv heads, head_dim), GQA
LOOP_SHAPES = [(64, 64, 128), (256, 64, 64)]           # 1536 work items per row: the block-stride loop


def _cabi():
    from lookaheaddecoding_b200 import _cabi
    return _cabi


def _fn(dtype):
    lib = _cabi().load()
    return lib.lade_rope_append_qknorm if dtype == torch.bfloat16 else lib.lade_rope_append_qknorm_f16


def _gen(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


def _is_canary(t):
    return bool((t == CANARY).all())


class Step:
    """One launch with canary-filled outputs: q_out [nh, q_pad, D]; each cache one flat buffer with 8 canary rows behind
    the last head's slab."""

    def __init__(self, dtype, nh, nkv, D, qkv, pos, wq, wk, eps=EPS, q_pad=None, cap=None, kv_len=5, max_pos=4096,
                 theta=1e6, call=None):
        cabi = _cabi()
        rows = qkv.shape[0]
        self.nh, self.nkv, self.D, self.rows, self.kv_len = nh, nkv, D, rows, kv_len
        self.q_pad = q_pad or rows + 3
        self.cap = cap or kv_len + rows + 4
        self.cos, self.sin = LR.rope_tables(D, max_pos, theta, dtype, "cuda")
        self.meta = torch.zeros(cabi.META_INTS, dtype=torch.int32, device="cuda")
        self.meta[cabi.M_KV_LEN] = kv_len
        self.qo = torch.full((nh, self.q_pad, D), CANARY, dtype=dtype, device="cuda")
        self.kbuf = torch.full(((nkv * self.cap + 8) * D,), CANARY, dtype=dtype, device="cuda")
        self.vbuf = torch.full(((nkv * self.cap + 8) * D,), CANARY, dtype=dtype, device="cuda")
        args = dict(stream=torch.cuda.current_stream().cuda_stream, qkv=qkv.data_ptr(), cos=self.cos.data_ptr(),
                    sin=self.sin.data_ptr(), pos=pos.data_ptr(), meta=self.meta.data_ptr(), q_out=self.qo.data_ptr(),
                    k=self.kbuf.data_ptr(), v=self.vbuf.data_ptr(), rows=rows, q_pad=self.q_pad, nh=nh, nkv=nkv, D=D,
                    cap=self.cap, max_pos=max_pos, wq=wq.data_ptr() if wq is not None else 0,
                    wk=wk.data_ptr() if wk is not None else 0, eps=eps)
        args.update(call or {})
        self.rc = _fn(dtype)(*args.values())
        torch.cuda.synchronize()
        self.kc = self.kbuf[: nkv * self.cap * D].view(nkv, self.cap, D)
        self.vc = self.vbuf[: nkv * self.cap * D].view(nkv, self.cap, D)
        self.pos = pos.long().clamp(0, max_pos - 1)

    def candidates(self, x, w, dtype):
        """[4, H, rows, D] for x [rows, H, D]."""
        return Q.candidates(x.transpose(0, 1), w, EPS, self.cos[self.pos], self.sin[self.pos], dtype)


def _split(qkv, nh, nkv, D):
    rows = qkv.shape[0]
    v = qkv.view(rows, nh + 2 * nkv, D)
    return v[:, :nh], v[:, nh:nh + nkv], v[:, nh + nkv:]


def _qkv(rows, nh, nkv, D, dtype, seed):
    g = _gen(seed)
    x = Q.data(rows, nh + 2 * nkv, D, dtype, g, "cuda").reshape(rows, -1).contiguous()
    return x, Q.weights(D, dtype, g, "cuda"), Q.weights(D, dtype, g, "cuda")


@pytest.mark.parametrize("dtn", list(DTYPES))
@pytest.mark.parametrize("nh,nkv,D", SHAPES + LOOP_SHAPES)
def test_position_zero_is_the_norm_itself(nh, nkv, D, dtn):
    dtype = DTYPES[dtn]
    rows = 37
    qkv, wq, wk = _qkv(rows, nh, nkv, D, dtype, nh + D)
    s = Step(dtype, nh, nkv, D, qkv, torch.zeros(rows, dtype=torch.int32, device="cuda"), wq, wk)
    assert s.rc == 0
    xq, xk, xv = _split(qkv, nh, nkv, D)
    took = 0
    for got, x, w in ((s.qo[:, :rows], xq, wq), (s.kc[:, s.kv_len:s.kv_len + rows], xk, wk)):
        main, alt = Q.norm_candidates(x.transpose(0, 1), w, EPS, dtype)
        bad, used = LR.unexplained(got, main, alt)
        assert bad == 0, f"{bad} elements are neither rounding of the float64 norm"
        took += used
    assert torch.equal(s.vc[:, s.kv_len:s.kv_len + rows], xv.transpose(0, 1))
    print(f"{dtn} {nh}/{nkv}/{D}: {took} elements took the rounding alternative")


@pytest.mark.parametrize("dtn", list(DTYPES))
@pytest.mark.parametrize("nh,nkv,D", SHAPES + LOOP_SHAPES)
def test_every_position_is_rope_of_a_norm_candidate(nh, nkv, D, dtn):
    dtype = DTYPES[dtn]
    rows = 120
    qkv, wq, wk = _qkv(rows, nh, nkv, D, dtype, 3 * nh + D)
    pos = torch.randint(0, 4096, (rows,), generator=_gen(1), device="cuda").to(torch.int32)
    s = Step(dtype, nh, nkv, D, qkv, pos, wq, wk)
    assert s.rc == 0
    xq, xk, xv = _split(qkv, nh, nkv, D)
    for got, x, w in ((s.qo[:, :rows], xq, wq), (s.kc[:, s.kv_len:s.kv_len + rows], xk, wk)):
        cands = s.candidates(x, w, dtype)
        assert Q.unexplained(got, cands) == 0
        # the weights matter: the other head type's weight explains almost nothing
        assert Q.unexplained(got, s.candidates(x, wk if w is wq else wq, dtype)) > got.numel() // 2
    assert torch.equal(s.vc[:, s.kv_len:s.kv_len + rows], xv.transpose(0, 1))
    assert _is_canary(s.qo[:, rows:])


@pytest.mark.parametrize("dtn", list(DTYPES))
@pytest.mark.parametrize("nh,nkv,D", SHAPES)
def test_zero_huge_and_extreme_rows(nh, nkv, D, dtn):
    dtype = DTYPES[dtn]
    rows = 8
    qkv, wq, wk = _qkv(rows, nh, nkv, D, dtype, 11)
    qkv[0] = 0
    huge = 1e18 if dtype == torch.bfloat16 else 6e4
    qkv[1, ::D] = huge                                   # one huge element in every head of the row
    qkv[2, :] = huge * 0.5
    if dtype == torch.float16:                            # rows near +-60000
        qkv[3] = (torch.rand(qkv.shape[1], generator=_gen(5), device="cuda") * 5e3 + 5.5e4).to(dtype)
        qkv[4] = -qkv[3]
        qkv[5, ::2] = 6e4
        qkv[5, 1::2] = -6e4
    pos = torch.tensor([0, 1, 7, 100, 1000, 4095, 3, 2], dtype=torch.int32, device="cuda")
    s = Step(dtype, nh, nkv, D, qkv, pos, wq, wk)
    assert s.rc == 0
    xq, xk, _ = _split(qkv, nh, nkv, D)
    for got, x, w in ((s.qo[:, :rows], xq, wq), (s.kc[:, s.kv_len:s.kv_len + rows], xk, wk)):
        assert torch.isfinite(got).all()
        assert bool((got[:, 0] == 0).all()), "a row of zeros must give zeros"
        assert Q.unexplained(got, s.candidates(x, w, dtype)) == 0


@pytest.mark.parametrize("dtn", list(DTYPES))
@pytest.mark.parametrize("over", [0, 5])
@pytest.mark.parametrize("nh,nkv,D", SHAPES + [(64, 8, 128)])
def test_clamped_positions_capacity_and_canaries(nh, nkv, D, over, dtn):
    """`over` rows of the step do not fit the cache: they are dropped, not written past the head's slab."""
    dtype = DTYPES[dtn]
    rows, q_pad, max_pos, kv_len = 37, 40, 512, 61
    qkv, wq, wk = _qkv(rows, nh, nkv, D, dtype, nh + D + over)
    pos = torch.randint(0, max_pos, (rows,), generator=_gen(over), device="cuda").to(torch.int32)
    qkv[1] = qkv[0]
    qkv[3] = qkv[4] = qkv[2]
    pos[:6] = torch.tensor([-3, 0, max_pos - 1, max_pos, max_pos + 7, -2 ** 31], dtype=torch.int32, device="cuda")
    s = Step(dtype, nh, nkv, D, qkv, pos, wq, wk, q_pad=q_pad, cap=kv_len + rows - over, kv_len=kv_len,
             max_pos=max_pos)
    assert s.rc == 0
    xq, xk, xv = _split(qkv, nh, nkv, D)
    assert Q.unexplained(s.qo[:, :rows], s.candidates(xq, wq, dtype)) == 0, "Q is incomplete or wrong"
    qo, kc, vc = s.qo, s.kc, s.vc
    assert torch.equal(qo[:, 0], qo[:, 1]) and torch.equal(qo[:, 2], qo[:, 3]) and torch.equal(qo[:, 2], qo[:, 4])
    assert torch.equal(kc[:, kv_len], kc[:, kv_len + 1]) and torch.equal(kc[:, kv_len + 2], kc[:, kv_len + 4])
    assert _is_canary(qo[:, rows:]), "pad rows of q_out were written"
    fit = rows - over
    assert Q.unexplained(kc[:, kv_len:], s.candidates(xk, wk, dtype)[:, :, :fit]) == 0
    assert torch.equal(vc[:, kv_len:], xv.transpose(0, 1)[:, :fit]), "V is not the input, bit for bit"
    assert _is_canary(kc[:, :kv_len]) and _is_canary(vc[:, :kv_len]), "a dropped row landed in the next head's slab"
    assert _is_canary(s.kbuf[nkv * s.cap * D:]) and _is_canary(s.vbuf[nkv * s.cap * D:]), \
        "a dropped row landed past the cache"


@pytest.mark.parametrize("dtn", list(DTYPES))
def test_argument_errors_write_nothing(dtn):
    cabi = _cabi()
    dtype = DTYPES[dtn]
    nh, nkv, D, rows = 8, 2, 128, 4
    qkv, wq, wk = _qkv(rows, nh, nkv, D, dtype, 0)
    pos = torch.zeros(rows, dtype=torch.int32, device="cuda")
    wide = torch.ones(2 * D, dtype=dtype, device="cuda")
    bad = [dict(wq=0), dict(wk=0), dict(eps=-1e-6), dict(eps=float("nan")), dict(eps=float("inf")),
           dict(wq=wide.data_ptr() + 2), dict(wk=wide.data_ptr() + 8), dict(qkv=0), dict(q_out=0), dict(rows=0),
           dict(q_pad=rows - 1), dict(D=72), dict(D=96), dict(D=528), dict(nh=0), dict(nkv=0)]
    for change in bad:
        s = Step(dtype, nh, nkv, D, qkv, pos, wq, wk, call=change)
        assert s.rc == cabi.LADE_EINVAL, f"{change}: rc {s.rc}"
        assert _is_canary(s.qo) and _is_canary(s.kbuf) and _is_canary(s.vbuf), f"{change}: something was written"
    assert Step(dtype, nh, nkv, D, qkv, pos, wq, wk, eps=0.0).rc == 0
