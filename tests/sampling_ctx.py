"""A bare context for launching the sampling verification kernels directly (``lade_sample_verify`` / ``_warped``).

The kernels read from a context only the guess tokens, ``S_DONE``, ``S_N_OLD`` and the old tokens, so
``lade_ctx_create`` + ``lade_ctx_reset`` at the target (W, N, G), with a configured vocabulary of 4096 to keep the pool
table small, serves launches on rows of any vocabulary (a per-launch argument).  Used by
``test_gpu_sampling_chain.py`` and ``tools/sampling_chain_cost.py``."""
import ctypes as C

import numpy as np
import torch

import state_scale as SS
from helpers import make_lade_config
from test_gpu_sampling_kernel import _DevInts, _Dims

CFG_VOCAB = 4096
EOS = CFG_VOCAB + 1


class Bare:
    """A context of shape (W, N, G) and its launch buffers."""

    def __init__(self, W, N, G):
        from lookaheaddecoding_b200 import _cabi
        self.C, self.lib = _cabi, _cabi.load()
        self.W, self.N, self.G, self.GS, self.WCAP = W, N, G, N - 1, W + N - 3
        self.R = 3 + self.GS + self.WCAP
        self.REC = self.R + 4 + W
        cfg = make_lade_config(W, N, G, CFG_VOCAB, 64 + 64 + N + 8, pool=True, eos=[EOS])
        self.ctx = C.c_void_p()
        self.C.check(self.lib.lade_ctx_create(C.byref(cfg), C.byref(self.ctx)), "create")
        prompt = [(7 * i) % 4000 + 20 for i in range(64)]
        pr, w0 = np.asarray(prompt, dtype=np.int32), np.asarray(SS.window0(prompt, self.WCAP, 0), dtype=np.int32)
        self.stream = torch.cuda.current_stream().cuda_stream
        self.C.check(self.lib.lade_ctx_reset(self.ctx, self.stream, pr.ctypes.data, len(pr), w0.ctypes.data, self.WCAP,
                                             64 + 64), "reset")
        torch.cuda.synchronize()
        fields = [("cfg", _cabi.LadeConfig), ("d", _Dims), ("state", C.c_void_p)]
        c = type("_Ctx", (C.Structure,), {"_fields_": fields}).from_address(self.ctx.value)
        self.d = c.d
        assert (self.d.W, self.d.N, self.d.G, self.d.GS, self.d.WCAP) == (W, N, G, self.GS, self.WCAP)
        self.st = torch.as_tensor(_DevInts(c.state, int(self.d.total_ints)), device="cuda")
        self.n_rows = 1 + self.WCAP + G * self.GS
        self.am = torch.randint(20, 4000, (self.n_rows,), dtype=torch.int32, device="cuda")
        self.rng = torch.zeros(2, dtype=torch.int64, device="cuda")
        self.n_dbg = 1 + (1 + G * self.GS + W)                    # count + the most draws one launch can make
        self.dbg = torch.zeros(self.n_dbg, dtype=torch.float32, device="cuda")

    def close(self):
        self.lib.lade_ctx_destroy(self.ctx)

    def meta(self, n_guess_tok):
        m = torch.zeros(self.C.META_INTS, dtype=torch.int32)
        m[self.C.M_PHASE] = 2 if n_guess_tok else 1
        m[self.C.M_TINY] = self.W
        m[self.C.M_N_GUESS_TOK] = n_guess_tok
        return m.cuda()

    def set_guess(self, tokens):
        assert len(tokens) % self.GS == 0 and len(tokens) // self.GS <= self.G
        self.st[self.d.off_guess:self.d.off_guess + len(tokens)] = torch.as_tensor(np.asarray(tokens, dtype=np.int32)).cuda()
        return self.meta(len(tokens))

    def launch(self, dtype, logits, vocab, meta, T, top_k=0, top_p=1.0, cuts=None, seed=0, offset=0, dbg=True,
               dbg_cuts=None):
        """cuts = None: lade_sample_verify; else (min_p, epsilon, eta) on lade_sample_verify_warped, which writes
        [rows visited, (threshold key, S') per row] to the float tensor dbg_cuts when one is given."""
        rec = torch.full((self.REC,), -7, dtype=torch.int32, device="cuda")
        self.rng.copy_(torch.tensor([seed, offset], dtype=torch.int64))
        sfx = "" if dtype == torch.bfloat16 else "_f16"
        dp = self.dbg.data_ptr() if dbg else 0
        if cuts is None:
            rc = getattr(self.lib, "lade_sample_verify" + sfx)(
                self.ctx, self.stream, logits.data_ptr(), logits.shape[1], vocab, self.am.data_ptr(), meta.data_ptr(),
                float(T), int(top_k), float(top_p), self.rng.data_ptr(), rec.data_ptr(), dp)
        else:
            w = self.C.LadeWarpers(float(T), int(top_k), float(top_p), *[float(c) for c in cuts])
            rc = getattr(self.lib, "lade_sample_verify_warped" + sfx)(
                self.ctx, self.stream, logits.data_ptr(), logits.shape[1], vocab, self.am.data_ptr(), meta.data_ptr(),
                C.byref(w), self.rng.data_ptr(), rec.data_ptr(), dp, 0 if dbg_cuts is None else dbg_cuts.data_ptr())
        self.C.check(rc, "sample verify")
        return rec.cpu().tolist()

    def exported(self):
        d = self.dbg.cpu().numpy()
        n = int(d[0])
        assert n <= self.n_dbg - 1
        return d[1:1 + n]


def device_logits(dtype, rows, ld, pad):
    rows = np.atleast_2d(rows)
    full = np.full((rows.shape[0], ld), pad, dtype=np.float64)
    full[:, :rows.shape[1]] = rows
    return torch.tensor(full, dtype=torch.float32).to(dtype).cuda()
