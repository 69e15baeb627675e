"""lade_rope_append_bias (Qwen2's q/k/v projection biases added to the fp32 projection, fused into RoPE + KV append)
against the host restatement of tests/qkv_bias_oracle.rope_bias: x = T(acc + float(b)) in fp32, then the rotary
embedding with every op rounded to the model dtype, V appended as x.  In bf16 and fp16, at head_dim 128 and 64, GQA:

* every element bit for bit, random positions, including more than 1024 work items per row (the loop path);
* exact integer probes (position 0, so RoPE is the identity): acc a row index, the bias nonzero on one head at a time
  and equal to the element's index in the head, plus one; acc + b is an exact integer, so a bias slice read from the
  wrong head, half or 8-element slice shows as a wrong integer;
* the rounding point: where T(T(acc) + b) != T(acc + b) the kernel gives the second (HF's addmm);
* a step that crosses kv_capacity, with canaries around the caches and behind q_out's rows;
* every argument error returns LADE_EINVAL and writes nothing.
"""
import pytest
import torch

import qkv_bias_oracle as B
from oracle import llama_ref as LR

pytestmark = pytest.mark.gpu
DTYPES = {"bf16": torch.bfloat16, "fp16": torch.float16}
CANARY = 777.0
SHAPES = [(8, 2, 128), (8, 4, 64), (28, 4, 128)]        # (q heads, kv heads, head_dim), GQA; the last Qwen2.5-7B's
LOOP_SHAPES = [(64, 64, 128), (256, 64, 64)]            # 1536 work items per row: the block-stride loop


def _cabi():
    from lookaheaddecoding_b200 import _cabi
    return _cabi


def _fn(dtype):
    lib = _cabi().load()
    return lib.lade_rope_append_bias if dtype == torch.bfloat16 else lib.lade_rope_append_bias_f16


def _gen(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


def _is_canary(t):
    return bool((t == CANARY).all())


class Step:
    """One launch with canary-filled outputs: q_out [nh, q_pad, D]; each cache one flat buffer with 8 canary rows behind
    the last head's slab."""

    def __init__(self, dtype, nh, nkv, D, acc, bias, pos, q_pad=None, cap=None, kv_len=5, max_pos=4096, theta=1e6,
                 call=None):
        cabi = _cabi()
        rows = acc.shape[0]
        self.rows, self.kv_len = rows, kv_len
        self.q_pad = q_pad or rows + 3
        self.cap = cap or kv_len + rows + 4
        self.cos, self.sin = LR.rope_tables(D, max_pos, theta, dtype, "cuda")
        self.meta = torch.zeros(cabi.META_INTS, dtype=torch.int32, device="cuda")
        self.meta[cabi.M_KV_LEN] = kv_len
        self.qo = torch.full((nh, self.q_pad, D), CANARY, dtype=dtype, device="cuda")
        self.kbuf = torch.full(((nkv * self.cap + 8) * D,), CANARY, dtype=dtype, device="cuda")
        self.vbuf = torch.full(((nkv * self.cap + 8) * D,), CANARY, dtype=dtype, device="cuda")
        args = dict(stream=torch.cuda.current_stream().cuda_stream, qkv=acc.data_ptr(), cos=self.cos.data_ptr(),
                    sin=self.sin.data_ptr(), pos=pos.data_ptr(), meta=self.meta.data_ptr(), q_out=self.qo.data_ptr(),
                    k=self.kbuf.data_ptr(), v=self.vbuf.data_ptr(), rows=rows, q_pad=self.q_pad, nh=nh, nkv=nkv, D=D,
                    cap=self.cap, max_pos=max_pos, bias=bias.data_ptr())
        args.update(call or {})
        self.rc = _fn(dtype)(*args.values())
        torch.cuda.synchronize()
        self.kc = self.kbuf[: nkv * self.cap * D].view(nkv, self.cap, D)
        self.vc = self.vbuf[: nkv * self.cap * D].view(nkv, self.cap, D)
        p = pos.long().clamp(0, max_pos - 1)
        self.want = B.rope_bias(acc, bias, nh, nkv, D, self.cos[p], self.sin[p], dtype)


def _data(rows, nh, nkv, D, dtype, seed, bias_scale=1.0):
    """fp32 projection rows (heads of their own scale, 1e-3 to 10) and a bias of about that size."""
    g = _gen(seed)
    C = (nh + 2 * nkv) * D
    acc = torch.randn(rows, nh + 2 * nkv, D, generator=g, device="cuda")
    acc = (acc * torch.exp(torch.empty(rows, nh + 2 * nkv, 1, device="cuda").uniform_(-6.9, 2.3, generator=g)))
    bias = (torch.randn(C, generator=g, device="cuda") * bias_scale).to(dtype)
    return acc.reshape(rows, C).contiguous(), bias


def _check_bits(s, rows, kv_len, fit=None):
    fit = rows if fit is None else fit
    q, k, v = s.want
    assert torch.equal(s.qo[:, :rows], q), "Q differs from the restatement"
    assert torch.equal(s.kc[:, kv_len:kv_len + fit], k[:, :fit]), "K differs from the restatement"
    assert torch.equal(s.vc[:, kv_len:kv_len + fit], v[:, :fit]), "V differs from the restatement"
    assert _is_canary(s.qo[:, rows:]), "pad rows of q_out were written"


@pytest.mark.parametrize("dtn", list(DTYPES))
@pytest.mark.parametrize("nh,nkv,D", SHAPES + LOOP_SHAPES)
def test_every_element_bit_for_bit(nh, nkv, D, dtn):
    dtype = DTYPES[dtn]
    rows = 120
    acc, bias = _data(rows, nh, nkv, D, dtype, nh + D)
    pos = torch.randint(0, 4096, (rows,), generator=_gen(1), device="cuda").to(torch.int32)
    s = Step(dtype, nh, nkv, D, acc, bias, pos)
    assert s.rc == 0
    _check_bits(s, rows, s.kv_len)
    assert _is_canary(s.kc[:, :s.kv_len]) and _is_canary(s.kc[:, s.kv_len + rows:])


@pytest.mark.parametrize("dtn", list(DTYPES))
@pytest.mark.parametrize("nh,nkv,D", SHAPES)
def test_integer_probes_one_head_at_a_time(nh, nkv, D, dtn):
    """acc[r, c] = r, bias = j + 1 at element j of head `hb` and 0 elsewhere, position 0: every output is the exact
    integer r (+ j + 1 on head hb)."""
    dtype = DTYPES[dtn]
    rows = 40
    nheads = nh + 2 * nkv
    acc = torch.arange(rows, dtype=torch.float32, device="cuda")[:, None].expand(rows, nheads * D).contiguous()
    pos = torch.zeros(rows, dtype=torch.int32, device="cuda")
    j = torch.arange(D, device="cuda", dtype=torch.float32)
    r = torch.arange(rows, device="cuda", dtype=torch.float32)[:, None]
    for hb in range(nheads):
        bias = torch.zeros(nheads, D, device="cuda")
        bias[hb] = j + 1
        bias = bias.reshape(-1).to(dtype)
        s = Step(dtype, nh, nkv, D, acc, bias, pos)
        assert s.rc == 0
        got = torch.cat([s.qo[:, :rows], s.kc[:, s.kv_len:s.kv_len + rows], s.vc[:, s.kv_len:s.kv_len + rows]])
        want = r.expand(rows, D)[None].repeat(nheads, 1, 1)
        want[hb] += j + 1
        bad = (got.float() != want).nonzero()
        assert bad.numel() == 0, f"bias on head {hb}: {len(bad)} wrong integers, first (head, row, elem) {bad[:4].tolist()}"


@pytest.mark.parametrize("dtn", list(DTYPES))
@pytest.mark.parametrize("nh,nkv,D", SHAPES[:2])
def test_rounding_point_is_hfs(nh, nkv, D, dtn):
    """The restatement that rounds twice, T(T(acc) + b), disagrees with the single rounding on many elements here; the
    kernel takes the single rounding on every one of them.  At position 0 the output is x itself."""
    dtype = DTYPES[dtn]
    rows = 64
    acc, bias = _data(rows, nh, nkv, D, dtype, 7, bias_scale=3.0)
    acc = torch.randn(acc.shape, generator=_gen(8), device="cuda")                     # one scale: about bias's
    pos = torch.zeros(rows, dtype=torch.int32, device="cuda")
    s = Step(dtype, nh, nkv, D, acc, bias, pos)
    assert s.rc == 0
    once = B.biased(acc, bias, dtype)
    twice = B.biased(acc.to(dtype).float(), bias, dtype)
    differ = once != twice
    got = torch.cat([s.qo[:, :rows], s.kc[:, s.kv_len:s.kv_len + rows], s.vc[:, s.kv_len:s.kv_len + rows]])
    got = got.transpose(0, 1).reshape(rows, -1)
    n = int(differ.sum())
    print(f"{dtn} {nh}/{nkv}/{D}: {n} of {differ.numel()} elements round differently when rounded twice")
    assert n > 100
    assert torch.equal(got, once)
    assert not (got[differ] == twice[differ]).any()


@pytest.mark.parametrize("dtn", list(DTYPES))
@pytest.mark.parametrize("over", [0, 5])
@pytest.mark.parametrize("nh,nkv,D", SHAPES[:2] + [(64, 8, 128)])
def test_capacity_clamped_positions_and_canaries(nh, nkv, D, over, dtn):
    """`over` rows of the step do not fit the cache: they are dropped, not written past the head's slab."""
    dtype = DTYPES[dtn]
    rows, q_pad, max_pos, kv_len = 37, 40, 512, 61
    acc, bias = _data(rows, nh, nkv, D, dtype, nh + D + over)
    pos = torch.randint(0, max_pos, (rows,), generator=_gen(over), device="cuda").to(torch.int32)
    pos[:6] = torch.tensor([-3, 0, max_pos - 1, max_pos, max_pos + 7, -2 ** 31], dtype=torch.int32, device="cuda")
    s = Step(dtype, nh, nkv, D, acc, bias, pos, q_pad=q_pad, cap=kv_len + rows - over, kv_len=kv_len, max_pos=max_pos)
    assert s.rc == 0
    _check_bits(s, rows, kv_len, fit=rows - over)
    assert _is_canary(s.kc[:, :kv_len]) and _is_canary(s.vc[:, :kv_len]), "a dropped row landed in the next head's slab"
    assert _is_canary(s.kbuf[nkv * s.cap * D:]) and _is_canary(s.vbuf[nkv * s.cap * D:]), \
        "a dropped row landed past the cache"


@pytest.mark.parametrize("dtn", list(DTYPES))
def test_argument_errors_write_nothing(dtn):
    cabi = _cabi()
    dtype = DTYPES[dtn]
    nh, nkv, D, rows = 8, 2, 128, 4
    acc, bias = _data(rows, nh, nkv, D, dtype, 0)
    pos = torch.zeros(rows, dtype=torch.int32, device="cuda")
    bad = [dict(bias=0), dict(bias=bias.data_ptr() + 2), dict(bias=bias.data_ptr() + 8), dict(qkv=acc.data_ptr() + 4),
           dict(qkv=0), dict(q_out=0), dict(rows=0), dict(q_pad=rows - 1), dict(D=72), dict(D=528), dict(nh=0),
           dict(nkv=0)]
    for change in bad:
        s = Step(dtype, nh, nkv, D, acc, bias, pos, call=change)
        assert s.rc == cabi.LADE_EINVAL, f"{change}: rc {s.rc}"
        assert _is_canary(s.qo) and _is_canary(s.kbuf) and _is_canary(s.vbuf), f"{change}: something was written"


def test_hf_linear_rounds_once():
    """What the kernel restates is what HF computes: nn.Linear with a bias on CUDA (Qwen2's q_proj) equals the fp32
    projection plus the bias rounded once, and both lie within the float64 bound with the bias term."""
    g = _gen(3)
    for dtype in DTYPES.values():
        x = torch.randn(120, 1024, generator=g, device="cuda").to(dtype)
        w = (torch.randn(1536, 1024, generator=g, device="cuda") * 0.03).to(dtype)
        b = (torch.randn(1536, generator=g, device="cuda") * 3).to(dtype)
        hf = torch.nn.functional.linear(x, w, b)
        acc = torch.mm(x, w.t(), out_dtype=torch.float32)
        once, twice = B.biased(acc, b, dtype), B.biased(acc.to(dtype).float(), b, dtype)
        ref, bound = B.linear_fp64(x, w, dtype, b)
        for name, y in (("HF", hf), ("fp32 mm + bias", once)):
            ok, mx, mean = LR.within_bound(y, ref, bound, mean_ratio=LR.LINEAR_MEAN_RATIO)
            print(f"{dtype} {name}: max ratio {mx:.3f} mean {mean:.3f}")
            assert ok, (dtype, name, mx, mean)
        agree_once = float((hf == once).float().mean())
        agree_twice = float((hf == twice).float().mean())
        print(f"{dtype}: HF equals the single rounding on {agree_once:.4f}, the double rounding on {agree_twice:.4f}")
        assert agree_once > agree_twice
