"""The wgmma attention kernel (impl 2 and the reference-order impl 3) must keep every output bit of the recorded build.

tests/golden/attn_bits.json holds the SHA-256 of lade_attn_fwd(_f16)'s output for the seeded cases of
tests/golden/gen_golden_attn_bits.py: the bench's steady shape at kv 1024 and 1278 with 4 splits, 40 heads with 3
splits, 1, 3 and 5 splits, a ring that wraps, GQA, a prefill of three q tiles, a lookahead-parallel rank (level and
dist offsets) and q <= 64 rows; bf16 and fp16.  Launch shape, split merge and pipelining may change; the arithmetic
(tiles, MMA operands, softmax update order, merge order) may not."""
import importlib.util
import json
import os

import pytest

from helpers import GOLD

pytestmark = pytest.mark.gpu

_spec = importlib.util.spec_from_file_location("gen_golden_attn_bits", os.path.join(GOLD, "gen_golden_attn_bits.py"))
GEN = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(GEN)
with open(os.path.join(GOLD, "attn_bits.json")) as _f:
    WANT = json.load(_f)["sha256"]


def test_every_case_is_recorded():
    assert sorted(WANT) == sorted(f"{n}/impl{i}/{d}" for n, i, d in GEN.keys())


@pytest.mark.parametrize("name,impl,dtype", list(GEN.keys()))
def test_attention_output_bits_unchanged(name, impl, dtype):
    assert GEN.run_case(name, impl, dtype) == WANT[f"{name}/impl{impl}/{dtype}"]
