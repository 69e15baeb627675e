// Device-resident lookahead decode state: 2-D window, n-gram pool, token buffers; the step-layout
// kernel and the fused verify / accept / pool-update kernel.
//
// Reference semantics (file:line into the reference checkout):
//   window init / fill / shift      lade/decoding.py:902, :1038-1066, :1119-1124
//   n-gram pool LRU                 lade/decoding.py:37-63, :80-96, :104-122
//   pool lookup for guesses         lade/decoding.py:948-954
//   step rows + position ids        lade/models/modeling_llama.py:1458-1511
//   mask scalars                    lade/models/modeling_llama.py:132-138
//   longest-prefix accept           lade/decoding.py:1071-1084
//   emission / EOS / stopping       lade/decoding.py:1165-1177, :1205-1219
#include "state.cuh"

#include <cstring>
#include <new>
#include <string>

namespace lade {

static thread_local std::string g_last_error;
void set_cuda_error(cudaError_t e, const char* where) {
  g_last_error = std::string(where) + ": " + cudaGetErrorString(e);
}
void set_error_string(const char* msg) { g_last_error = msg; }

// One LRU insertion into the pool, executed cooperatively by one warp (all 32 lanes call it).
// `tup` points at GS ints readable by every lane.  lade/decoding.py:39-49.
__device__ void pool_insert_warp(int* st, const Dims& d, int key, const int* tup) {
  const int lane = threadIdx.x & 31;
  if (d.G <= 0 || key < 0 || key >= d.V) return;   // G = 0: no pool (and no slot to write: `last` would be -1)
  int* cnt = st + d.off_cnt;
  int* base = st + d.off_tup + (long long)key * d.G * d.GS;
  const int c = cnt[key];
  const int GS = d.GS;
  int found = -1;
  for (int g0 = 0; g0 < c && found < 0; g0 += 32) {
    const int g = g0 + lane;
    bool match = g < c;
    if (match) {
      for (int j = 0; j < GS; ++j) match = match && (base[g * GS + j] == tup[j]);
    }
    const unsigned b = __ballot_sync(0xffffffffu, match);
    if (b) found = g0 + __ffs(b) - 1;
  }
  int shift_from;  // entries [shift_from+1, c) move down by one slot
  int new_cnt = c;
  if (found >= 0) {
    shift_from = found;
  } else if (c < d.G) {
    shift_from = c;  // nothing to shift
    new_cnt = c + 1;
  } else {
    shift_from = 0;  // drop the oldest
  }
  const int last = (found >= 0 || c >= d.G) ? c - 1 : c;  // slot that receives the tuple
  const int lo = shift_from * GS, hi = last * GS;           // ints [lo, hi) take the value GS ahead
  for (int k = lo; k < hi; k += 32) {
    const int i = k + lane;
    int v = 0;
    if (i < hi) v = base[i + GS];
    __syncwarp();
    if (i < hi) base[i] = v;
    __syncwarp();
  }
  if (lane < GS) base[last * GS + lane] = tup[lane];
  if (lane == 0) cnt[key] = new_cnt;
  __syncwarp();
}

// ---- reset: pool from prompt ------------------------------------------------------------------
__global__ void fill_pool_from_prompt_kernel(int* st, Dims d, int n_prompt) {
  // Insertions with different keys touch disjoint pool rows; only the order WITHIN one key matters (LRU).
  // Every warp of the grid walks the prompt in order, 32 positions per ballot, and performs the insertions
  // whose key it owns (key % n_warps), lane-parallel inside one insertion -- P/n_warps serial steps per warp
  // instead of P on a single warp.
  __shared__ int tup_all[8][32];
  const int lane = threadIdx.x & 31;
  const int wib = threadIdx.x >> 5;
  const int n_warps = gridDim.x * (blockDim.x >> 5);
  const int me = blockIdx.x * (blockDim.x >> 5) + wib;
  int* tup = tup_all[wib];
  const int* ids = st + d.off_out;
  const int n_pos = n_prompt - d.N + 1;
  for (int s0 = 0; s0 < n_pos; s0 += 32) {
    const int s = s0 + lane;
    const int key = s < n_pos ? ids[s] : -1;
    unsigned mine = __ballot_sync(0xffffffffu, key >= 0 && (key % n_warps) == me);
    while (mine) {
      const int src = __ffs(mine) - 1;
      mine &= mine - 1;
      const int sk = s0 + src;
      if (lane < d.GS) tup[lane] = ids[sk + 1 + lane];
      __syncwarp();
      pool_insert_warp(st, d, ids[sk], tup);
    }
  }
}

__global__ void reset_header_kernel(int* st, Dims d, int n_prompt, int n_window0, int max_length) {
  const int t = threadIdx.x;
  if (t == 0) {
    st[S_FILL_LEVEL] = 0;
    st[S_LST_TOKEN] = -1;
    st[S_KV_LEN] = 0;
    st[S_N_OUT] = n_prompt;
    st[S_N_OLD] = n_prompt;
    st[S_DONE] = 0;
    st[S_STEPS] = 0;
    st[S_MAX_LENGTH] = max_length;
    st[S_N_PROMPT] = n_prompt;
    st[S_N_GUESS_TOK] = 0;
    st[S_SKIP] = 0;
  }
  if (t < d.N - 1) st[d.off_win_len + t] = (t == 0) ? n_window0 : 0;
  // all_old_tokens starts as a copy of the prompt (decoding.py:879)
  for (int i = t; i < n_prompt; i += blockDim.x) st[d.off_old + i] = st[d.off_out + i];
}

// ---- step layout -------------------------------------------------------------------------------
__global__ void step_layout_kernel(int* st, Dims d, int q_pad, int* ids_out, int* pos_out, int* rd_out,
                                   int* lm_rows, int* meta, unsigned* rowmask, int mask_words) {
  __shared__ int s_sizes[64];
  __shared__ int s_start[64];
  __shared__ int s_off[64];
  __shared__ int s_hdr[16];
  const int t = threadIdx.x;
  const int N = d.N, GS = d.GS;
  if (t == 0) {
    const int fill = st[S_FILL_LEVEL];
    const int* wl = st + d.off_win_len;
    int phase = (wl[1] == 0) ? 0 : ((wl[N - 2] == 0) ? 1 : 2);
    const int n_out = st[S_N_OUT];
    const int skip = st[S_SKIP];                                                        // decoding.py:941-942
    const int n_input = (phase == 0) ? n_out : 1 + skip;
    // lookahead parallelism: this rank owns window columns [ws, we) (decoding.py:973-984)
    int ws = 0, we = wl[0] + 1;
    if (d.D > 1) {
      const int window_len = wl[0] + 1;
      const int split = (window_len + d.D - 1) / d.D;
      ws = min(split * d.rank, window_len);
      we = min(split * (d.rank + 1), window_len);
    }
    int acc = n_input;
    for (int l = 0; l <= fill; ++l) {
      const int sz = (l == 0) ? max(we - 1, 0) : (d.D > 1 ? we - ws : wl[l]);
      s_sizes[l] = sz;
      s_off[l] = (l == 0 || d.D == 1) ? 0 : ws;
      s_start[l] = acc;
      acc += sz;
    }
    int n_ng = 0, g0 = 0;
    const int lst = st[S_LST_TOKEN];
    if (phase == 2 && lst >= 0 && lst < d.V && d.G > 0) n_ng = st[d.off_cnt + lst];     // decoding.py:948
    if (d.D > 1 && n_ng > 0) {                                                          // decoding.py:956-963
      const int per = (n_ng + d.D - 1) / d.D;
      g0 = min(per * d.rank, n_ng);
      n_ng = min(per * (d.rank + 1), n_ng) - g0;
    }
    const int lg = n_ng * GS;
    const int q_len = acc + lg;
    const int tiny = s_sizes[fill];
    const int level_offset = n_input - 1;                                               // modeling :136
    const int dist_offset = 1 + s_sizes[0] - tiny;                                      // modeling :137
    s_hdr[0] = phase; s_hdr[1] = n_input; s_hdr[2] = fill + 1; s_hdr[3] = lg; s_hdr[4] = q_len;
    s_hdr[5] = tiny; s_hdr[6] = level_offset; s_hdr[7] = level_offset + dist_offset;
    s_hdr[8] = n_out; s_hdr[9] = lst; s_hdr[10] = acc;  // acc = first guess row
    s_hdr[11] = g0 * GS;
    st[S_N_GUESS_TOK] = lg;
    meta[LADE_M_Q_LEN] = q_len;
    meta[LADE_M_KV_LEN] = st[S_KV_LEN];
    meta[LADE_M_N_INPUT] = n_input;
    meta[LADE_M_LEVEL_OFFSET] = level_offset;
    meta[LADE_M_ALL_OFFSET] = level_offset + dist_offset;
    meta[LADE_M_TINY] = tiny;
    meta[LADE_M_N_LEVELS] = fill + 1;
    meta[LADE_M_N_GUESS_TOK] = lg;
    meta[LADE_M_IS_PREFILL] = (phase == 0);
    meta[LADE_M_PHASE] = phase;
    meta[LADE_M_Q_PAD] = q_pad;
    meta[LADE_M_DONE] = st[S_DONE];
    meta[LADE_M_STEP] = st[S_STEPS];
  }
  __syncthreads();
  const int phase = s_hdr[0], n_input = s_hdr[1], n_levels = s_hdr[2], lg = s_hdr[3], q_len = s_hdr[4];
  const int tiny = s_hdr[5], a_off = s_hdr[7], n_out = s_hdr[8], lst = s_hdr[9], g_row0 = s_hdr[10];
  const int lst_id = n_out - 1;                                                         // modeling :1466
  const int* out_ids = st + d.off_out;
  const int* gsrc = st + d.off_tup + (long long)(lst < 0 ? 0 : lst) * d.G * GS + s_hdr[11];
  int* gdst = st + d.off_guess;
  for (int r = t; r < q_pad; r += blockDim.x) {
    int id = 0, pos = 0, rd = rowdesc_make(LADE_ROW_PAD, 0, 0);
    if (r < n_input) {
      id = out_ids[n_out - n_input + r];
      pos = lst_id - n_input + 1 + r;
    } else if (r < g_row0) {
      int l = 0;
      while (l + 1 < n_levels && r >= s_start[l + 1]) ++l;
      const int j = r - s_start[l];
      id = st_win(st, d, l)[s_off[l] + j];
      if (l == 0) pos = lst_id + 1 + j;                                                 // modeling :1494
      else pos = lst_id + l + (s_sizes[0] + 1 - s_sizes[l]) + j;                        // modeling :1496-1497
    } else if (r < q_len) {
      const int gi = r - g_row0;
      id = gsrc[gi];
      gdst[gi] = id;                       // remembered for the verification of this step
      pos = lst_id + 1 + (gi % GS);                                                     // modeling :1501
    }
    if (r < q_len) {
      if (phase == 0 || r < a_off) rd = rowdesc_make(LADE_ROW_PREFIX, 0, r & 0x7fff);
      else if (r < g_row0) rd = rowdesc_make(LADE_ROW_WINDOW, (r - a_off) / max(tiny, 1), (r - a_off) % max(tiny, 1));
      else rd = rowdesc_make(LADE_ROW_GUESS, (r - g_row0) / GS, (r - g_row0) % GS);
    }
    ids_out[r] = id;
    pos_out[r] = pos;
    rd_out[r] = rd;
  }
  // lm_head rows: slot 0 = next-token row, [1, 1+WCAP) newest window level, then verification rows
  for (int s = t; s < d.lm_cap; s += blockDim.x) {
    int row = n_input - 1;
    if (s >= 1 && s < 1 + d.WCAP) {
      const int i = s - 1;
      if (i < tiny) row = q_len - lg - tiny + i;                                        // modeling :1581-1591
    } else if (s >= 1 + d.WCAP) {
      const int i = s - 1 - d.WCAP;
      if (i < lg) row = q_len - lg + i;                                                 // modeling :1592
    }
    lm_rows[s] = row;
  }
  // Visibility bitmask of the step block, one row of `mask_words` words per query row: the attention
  // kernels test these bits in registers instead of re-deriving the predicate per head and per layer.
  if (rowmask != nullptr && phase != 0) {
    __syncthreads();                                  // rd_out of every row is written
    const int level_offset = s_hdr[6];
    for (int w = t; w < q_pad * mask_words; w += blockDim.x) {
      const int r = w / mask_words, wi = w % mask_words;
      unsigned bits = 0;
      if (r < q_len) {
        const int rd_r = rd_out[r];
        for (int i = 0; i < 32; ++i) {
          const int c = wi * 32 + i;
          if (c < q_len && row_sees(rd_r, r, rd_out[c], c, level_offset)) bits |= 1u << i;
        }
      }
      rowmask[w] = bits;
    }
  }
}

// ---- verify + accept + pool update ---------------------------------------------------------------
// A step's decision: what every rank must agree on before the state update.  Single GPU: computed and
// applied by one kernel.  Lookahead parallelism: each rank writes its local decision as a fixed-size
// int32 record, the records are all-gathered (one NCCL call), every rank reduces them identically.
//   record = [first_guess, max_hit, n_new, hits[GS], new_tokens[WCAP]]
struct Decision {
  int first_guess, max_hit, max_hit_idx, n_new;
  int sampling;        // sampling-path semantics of the emission loop (decoding.py:594-603)
  int extra_finished;  // host-evaluated stop condition (sampling path, decoding.py:636-643)
  int hits[64];
  int new_tok[1024 + 64];
  int filt[1024];      // sampling + EOS: newest window level after filter_window (decoding.py:131-135,578-580)
};


// Local part: argmax slots -> decision (longest-prefix accept over this rank's guesses, decoding.py:1071-1084).
__device__ void local_decision(int* st, const Dims& d, const int* __restrict__ am, const int* __restrict__ meta,
                               Decision* dec, int* s_best) {
  const int t = threadIdx.x;
  const int GS = d.GS, WCAP = d.WCAP;
  const int tiny = meta[LADE_M_TINY];
  const int lg = meta[LADE_M_N_GUESS_TOK];
  const int phase = meta[LADE_M_PHASE];
  const int first_guess = am[0];
  const int* inp = am + 1;
  const int* gres = am + 1 + WCAP;
  if (t == 0) { *s_best = 0; dec->first_guess = first_guess; dec->n_new = tiny; dec->sampling = 0; dec->extra_finished = 0; }
  if (t < GS) dec->hits[t] = (t == 0) ? first_guess : 0;
  for (int j = t; j < tiny; j += blockDim.x) dec->new_tok[j] = inp[j];
  __syncthreads();
  if (phase == 2) {
    const int n_ng = lg / GS;
    const int* gtok = st + d.off_guess;
    for (int e0 = 0; e0 < n_ng; e0 += blockDim.x) {
      const int e = e0 + t;
      if (e < n_ng) {
        int gg = GS - 1;
        for (int u = 0; u < GS; ++u) {
          const int correct = (u == 0) ? first_guess : gres[e * GS + u - 1];
          if (gtok[e * GS + u] != correct) { gg = u; break; }
        }
        if (gg > 0) atomicMax(s_best, gg * 65536 + (65535 - e));   // strictly longer wins, then earliest
      }
    }
    __syncthreads();
    const int best = *s_best;
    if (best > 0) {
      const int mh = best >> 16, e = 65535 - (best & 0xffff);
      if (t <= mh) dec->hits[t] = (t == 0) ? first_guess : gres[e * GS + t - 1];
    }
  }
  __syncthreads();
  if (t == 0) {
    const int best = *s_best;
    dec->max_hit = best >> 16;
    dec->max_hit_idx = best > 0 ? 65535 - (best & 0xffff) : 0;
  }
  __syncthreads();
}

// Reduce the D gathered records to the decision every rank applies (decoding.py:1023-1024,1043-1058,1088-1107).
__device__ void gathered_decision(const Dims& d, const int* __restrict__ recs, const int* __restrict__ meta, Decision* dec) {
  const int t = threadIdx.x;
  const int R = lp_rec_ints(d), GS = d.GS;
  const int phase = meta[LADE_M_PHASE];
  __shared__ int s_winner, s_base[65];
  if (t == 0) {
    dec->sampling = 0; dec->extra_finished = 0;
    dec->first_guess = recs[0];                          // rank 0's token (torch.distributed.broadcast src=0)
    int mh = 0, win = 0;
    for (int r = 0; r < d.D; ++r)
      if (recs[r * R + 1] > mh) { mh = recs[r * R + 1]; win = r; }      // list.index(max): first rank wins
    dec->max_hit = mh;
    dec->max_hit_idx = 0;
    s_winner = win;
    int acc = 0;
    for (int r = 0; r < d.D; ++r) { s_base[r] = acc; acc += recs[r * R + 2]; }
    s_base[d.D] = acc;
    dec->n_new = (phase == 0) ? recs[(d.D - 1) * R + 2] : acc;           // prefill: last rank holds all of L1
  }
  __syncthreads();
  if (t < GS) dec->hits[t] = dec->max_hit > 0 ? recs[s_winner * R + 3 + t] : (t == 0 ? dec->first_guess : 0);
  if (phase == 0) {
    const int* src = recs + (d.D - 1) * R + 3 + GS;
    for (int j = t; j < dec->n_new; j += blockDim.x) dec->new_tok[j] = src[j];
  } else {
    for (int r = 0; r < d.D; ++r) {
      const int n = recs[r * R + 2];
      const int* src = recs + r * R + 3 + GS;
      for (int j = t; j < n; j += blockDim.x) dec->new_tok[s_base[r] + j] = src[j];
    }
  }
  __syncthreads();
}

// Apply a decision: window fill/shift, pool update, emission, EOS, KV bookkeeping, result record.
__device__ void apply_decision(int* st, const Dims& d, const Decision* dec, const int* __restrict__ meta, int* res,
                               int* s_tup) {
  const int t = threadIdx.x;
  const int N = d.N, GS = d.GS, W = d.W;
  const int phase = meta[LADE_M_PHASE];
  const int n_input = meta[LADE_M_N_INPUT];
  const int q_len = meta[LADE_M_Q_LEN];
  const int lg = meta[LADE_M_N_GUESS_TOK];
  const int kv_len = st[S_KV_LEN];
  int* wl = st + d.off_win_len;
  const int fill = st[S_FILL_LEVEL];
  const int lst_token = st[S_LST_TOKEN];
  const int first_guess = dec->first_guess;
  const int n_new = dec->n_new;

  if (phase == 0) {                                                                     // decoding.py:1038-1048
    int* L0 = st_win(st, d, 0);
    const int len0 = wl[0];
    for (int j0 = 0; j0 < len0 - 1; j0 += blockDim.x) {
      const int j = j0 + t;
      int v = 0;
      if (j < len0 - 1) v = L0[j + 1];
      __syncthreads();
      if (j < len0 - 1) L0[j] = v;
      __syncthreads();
    }
    int* L1 = st_win(st, d, 1);
    for (int j = t; j < n_new; j += blockDim.x) L1[j] = dec->new_tok[j];
    __syncthreads();
    if (t == 0) { wl[0] = len0 - 1; wl[1] = n_new; st[S_FILL_LEVEL] = 1; }
  } else if (phase == 1) {                                                              // decoding.py:1049-1066
    for (int l = 0; l <= fill; ++l) {
      int* L = st_win(st, d, l);
      const int len = wl[l];
      for (int j0 = 0; j0 < len - 1; j0 += blockDim.x) {
        const int j = j0 + t;
        int v = 0;
        if (j < len - 1) v = L[j + 1];
        __syncthreads();
        if (j < len - 1) L[j] = v;
        __syncthreads();
      }
    }
    int* Ln = st_win(st, d, fill + 1);
    for (int j = t; j + 1 < n_new; j += blockDim.x) Ln[j] = dec->new_tok[j + 1];
    __syncthreads();
    if (t == 0) {
      for (int l = 0; l <= fill; ++l) wl[l] = wl[l] - 1;
      wl[fill + 1] = n_new - 1;
      st[S_FILL_LEVEL] = fill + 1;
    }
  } else {
    // ---- pool update with the pre-shift window (decoding.py:1116, :37-63)
    if (t < 32) {
      const int* L0 = st_win(st, d, 0);
      for (int i = 0; i < W; ++i) {
        const int key = (i == 0) ? lst_token : L0[i - 1];
        if (t < GS) s_tup[t] = (t < GS - 1) ? st_win(st, d, t + 1)[i] : dec->new_tok[i];
        __syncwarp();
        pool_insert_warp(st, d, key, s_tup);
      }
    }
    __syncthreads();
    // ---- window shift (decoding.py:1119-1124); levels are disjoint buffers, go bottom-up
    for (int l = 0; l < N - 2; ++l) {
      int* dst = st_win(st, d, l);
      const int* src = st_win(st, d, l + 1);
      const int off = (l == 0) ? 1 : 0;
      const int len = W - off;
      for (int j = t; j < len; j += blockDim.x) dst[j] = src[j + off];
      __syncthreads();
    }
    int* Llast = st_win(st, d, N - 2);
    for (int j = t; j < W; j += blockDim.x) Llast[j] = (dec->sampling & 2) ? dec->filt[j] : dec->new_tok[j];
    __syncthreads();
  }
  __syncthreads();

  // ---- emission, EOS scan, POOL_FROM_PROMPT appends, stopping (warp 0; decoding.py:1145-1219)
  if (t < 32) {
    const int max_hit = dec->max_hit;
    const int max_hit_idx = dec->max_hit_idx;
    const int kvcache_len = kv_len + n_input;                                           // modeling :1570
    // LP with a hit: no KV copy, the accepted tokens are re-fed next step (decoding.py:1148-1153)
    const bool refeed = (d.D > 1 && max_hit > 0);
    int n_old = st[S_N_OLD];
    int* old = st + d.off_old;
    int n_emit = max_hit + 1;
    bool finished = false;
    for (int h = 0; h <= max_hit; ++h) {
      if (d.n_eos > 0 && dec->hits[h] == d.eos[0]) {
        if (t == 0 && n_old < d.cap) old[n_old] = dec->hits[h];
        n_old++;
        n_emit = h + 1;
        finished = true;
        break;
      }
      // greedy path appends the LAST hit every time (sic, decoding.py:1175); the sampling path the right one (:601)
      if (t == 0 && n_old < d.cap) old[n_old] = (dec->sampling & 1) ? dec->hits[h] : dec->hits[max_hit];
      n_old++;
      __syncwarp();
      if (d.pool_from_prompt && n_old >= N && n_old <= d.cap) {                         // decoding.py:1176-1177
        if (t < GS) s_tup[t] = old[n_old - N + 1 + t];
        __syncwarp();
        pool_insert_warp(st, d, old[n_old - N], s_tup);
      }
    }
    if (!finished) {
      if (dec->sampling & 1) finished = dec->extra_finished != 0;
      else for (int k = 0; k < d.n_eos; ++k) finished = finished || (first_guess == d.eos[k]);  // :1205-1212
    }
    const int n_out = st[S_N_OUT];
    int* out = st + d.off_out;
    if (t < n_emit && n_out + t < d.cap) out[n_out + t] = dec->hits[t];
    __syncwarp();
    if (t == 0) {
      const int n_out_new = n_out + n_emit;
      const int done = (finished || n_out_new >= st[S_MAX_LENGTH]) ? 1 : 0;              // :1215-1219
      const int kv_new = refeed ? kvcache_len : kvcache_len + max_hit;
      st[S_N_OUT] = n_out_new;
      st[S_N_OLD] = n_old;
      st[S_KV_LEN] = kv_new;
      st[S_SKIP] = refeed ? max_hit : 0;
      st[S_LST_TOKEN] = dec->hits[max_hit];                                             // :1165
      st[S_DONE] = done;
      st[S_STEPS] = st[S_STEPS] + 1;
      res[LADE_R_N_EMIT] = n_emit;
      res[LADE_R_MAX_HIT] = max_hit;
      res[LADE_R_MAX_HIT_IDX] = max_hit_idx;
      res[LADE_R_KV_SRC] = (max_hit > 0 && !refeed) ? (kv_len + q_len - lg + max_hit_idx * GS) : -1;  // :1156
      res[LADE_R_KV_DST] = kvcache_len;
      res[LADE_R_KV_LEN] = kv_new;
      res[LADE_R_DONE] = done;
      res[LADE_R_N_OUT] = n_out_new;
      res[LADE_R_STEPS] = st[S_STEPS];
      res[LADE_R_N_GUESS] = lg / GS;
    }
    if (t < GS) res[LADE_R_HITS + t] = dec->hits[t];
  }
}

__device__ void write_done_result(int* st, int* res) {
  if (threadIdx.x == 0) {
    res[LADE_R_N_EMIT] = 0; res[LADE_R_DONE] = 1; res[LADE_R_MAX_HIT] = 0; res[LADE_R_KV_SRC] = -1;
    res[LADE_R_N_OUT] = st[S_N_OUT]; res[LADE_R_STEPS] = st[S_STEPS]; res[LADE_R_KV_LEN] = st[S_KV_LEN];
  }
}

__global__ void accept_update_kernel(int* st, Dims d, const int* __restrict__ am, const int* __restrict__ meta,
                                     int* res) {
  __shared__ Decision dec;
  __shared__ int s_tup[64];
  __shared__ int s_best;
  if (st[S_DONE]) { write_done_result(st, res); return; }
  local_decision(st, d, am, meta, &dec, &s_best);
  apply_decision(st, d, &dec, meta, res, s_tup);
}

// Externally decided step (sampling path: the host runs the reference's rejection-sampling verification,
// decoding.py:484-540, with the python/torch RNG streams): apply [record | max_hit_idx, flags, finished].
__global__ void commit_decision_kernel(int* st, Dims d, const int* __restrict__ rec, const int* __restrict__ meta, int* res) {
  __shared__ Decision dec;
  __shared__ int s_tup[64];
  const int t = threadIdx.x;
  if (st[S_DONE]) { write_done_result(st, res); return; }
  const int R = lp_rec_ints(d);
  if (t == 0) {
    dec.first_guess = rec[0]; dec.max_hit = rec[1]; dec.n_new = rec[2];
    dec.max_hit_idx = rec[R]; dec.sampling = rec[R + 1] & 3; dec.extra_finished = rec[R + 2];
  }
  if (rec[R + 1] & 2)
    for (int j = t; j < d.W; j += blockDim.x) dec.filt[j] = rec[R + 4 + j];
  if (t < d.GS) dec.hits[t] = rec[3 + t];
  for (int j = t; j < d.WCAP; j += blockDim.x) dec.new_tok[j] = rec[3 + d.GS + j];
  __syncthreads();
  apply_decision(st, d, &dec, meta, res, s_tup);
}

// LP, local half: write this rank's record.
__global__ void lp_verify_kernel(int* st, Dims d, const int* __restrict__ am, const int* __restrict__ meta, int* rec) {
  __shared__ Decision dec;
  __shared__ int s_best;
  const int t = threadIdx.x;
  if (st[S_DONE]) {
    for (int i = t; i < lp_rec_ints(d); i += blockDim.x) rec[i] = 0;
    return;
  }
  local_decision(st, d, am, meta, &dec, &s_best);
  if (t == 0) { rec[0] = dec.first_guess; rec[1] = dec.max_hit; rec[2] = dec.n_new; }
  if (t < d.GS) rec[3 + t] = dec.hits[t];
  for (int j = t; j < d.WCAP; j += blockDim.x) rec[3 + d.GS + j] = j < dec.n_new ? dec.new_tok[j] : 0;
}

// LP, global half: reduce the gathered records and update the (replicated) state.
__global__ void lp_commit_kernel(int* st, Dims d, const int* __restrict__ recs, const int* __restrict__ meta, int* res) {
  __shared__ Decision dec;
  __shared__ int s_tup[64];
  if (st[S_DONE]) { write_done_result(st, res); return; }
  gathered_decision(d, recs, meta, &dec);
  apply_decision(st, d, &dec, meta, res, s_tup);
}

// ---- KV compaction ---------------------------------------------------------------------------------
// grid: (n_layers * 2 * n_kv_heads, max_rows) ; block: head_dim/8 threads (16 B each)
__global__ void kv_compact_kernel(const int* __restrict__ res, __nv_bfloat16* k_base, __nv_bfloat16* v_base,
                                  long long layer_stride, int n_kv_heads, int kv_capacity, int head_dim) {
  const int max_hit = res[LADE_R_MAX_HIT];
  const int row = blockIdx.y;
  if (row >= max_hit) return;
  const int src = res[LADE_R_KV_SRC], dst = res[LADE_R_KV_DST];
  if (src < 0) return;
  const int idx = blockIdx.x;
  const int head = idx % n_kv_heads;
  const int kv = (idx / n_kv_heads) & 1;
  const int layer = idx / (2 * n_kv_heads);
  __nv_bfloat16* base = (kv ? v_base : k_base) + layer * layer_stride + (long long)head * kv_capacity * head_dim;
  const uint4* s = reinterpret_cast<const uint4*>(base + (long long)(src + row) * head_dim);
  uint4* dptr = reinterpret_cast<uint4*>(base + (long long)(dst + row) * head_dim);
  if (threadIdx.x * 8 < head_dim) dptr[threadIdx.x] = s[threadIdx.x];
}

// ---- row-wise argmax (lowest index on ties) ------------------------------------------------------------
// Argmax of row `row` into out_idx[row], by the whole CTA: 16-byte loads when the row is aligned, each element converted
// to fp32 and passed through `score(f, id)` (the identity for lade_argmax_rows, the logits processors for
// lade_argmax_processed) before it competes, then a lowest-index reduction over the block.  An all -inf row yields 0,
// like torch.argmax.
struct IdentityScore {
  __device__ __forceinline__ float operator()(float f, int) const { return f; }
};

template <typename T, typename Score>
__device__ __forceinline__ void argmax_row(const T* __restrict__ logits, int vocab, int ld, int row, Score score,
                                           int* out_idx) {
  const T* p = logits + (long long)row * ld;
  float best = -INFINITY;
  int bi = 0x7fffffff;
  const int t = threadIdx.x;
  const int nvec = vocab / 8;
  const uint4* pv = reinterpret_cast<const uint4*>(p);
  const bool aligned = ((reinterpret_cast<uintptr_t>(p) & 15) == 0);
  if (aligned) {
    for (int i = t; i < nvec; i += blockDim.x) {
      const uint4 v = pv[i];
      const T* e = reinterpret_cast<const T*>(&v);
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const float f = score(Elem<T>::to_f(e[j]), i * 8 + j);
        const int id = i * 8 + j;
        if (f > best || (f == best && id < bi)) { best = f; bi = id; }
      }
    }
    for (int id = nvec * 8 + t; id < vocab; id += blockDim.x) {
      const float f = score(Elem<T>::to_f(p[id]), id);
      if (f > best || (f == best && id < bi)) { best = f; bi = id; }
    }
  } else {
    for (int id = t; id < vocab; id += blockDim.x) {
      const float f = score(Elem<T>::to_f(p[id]), id);
      if (f > best || (f == best && id < bi)) { best = f; bi = id; }
    }
  }
  // NaN handling: torch.argmax treats NaN as maximal; random-init/finite models never produce it.
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float ob = __shfl_xor_sync(0xffffffffu, best, o);
    const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
    if (ob > best || (ob == best && oi < bi)) { best = ob; bi = oi; }
  }
  __shared__ float s_b[32];
  __shared__ int s_i[32];
  const int warp = t >> 5, lane = t & 31;
  if (lane == 0) { s_b[warp] = best; s_i[warp] = bi; }
  __syncthreads();
  if (warp == 0) {
    const int nw = blockDim.x >> 5;
    best = lane < nw ? s_b[lane] : -INFINITY;
    bi = lane < nw ? s_i[lane] : 0x7fffffff;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const float ob = __shfl_xor_sync(0xffffffffu, best, o);
      const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
      if (ob > best || (ob == best && oi < bi)) { best = ob; bi = oi; }
    }
    if (lane == 0) out_idx[row] = (bi == 0x7fffffff) ? 0 : bi;
  }
}

template <typename T>
__global__ void argmax_rows_kernel(const T* __restrict__ logits, int vocab, int ld, int* out_idx) {
  argmax_row(logits, vocab, ld, blockIdx.x, IdentityScore(), out_idx);
}

// ---- argmax under the greedy logits processors ----------------------------------------------------------
// Slot s of the lm rows is scored as HF's greedy step scores the position it stands for:
// argmax(processors(prefix, fp32(logits[s]))).  Prefix of slot 0: out_ids[0, n_out); of verification slot 1+WCAP+i
// (i < lg, n-gram e = i / GS, position u = i % GS): out_ids[0, n_out) + guess[e*GS .. e*GS+u] -- the columns row_sees
// gives that GUESS row.  Window slots (and verification slots past lg, which accept never reads) stay plain argmax.
// Each CTA marks its prefix's tokens in two V-bit shared bitmaps, "penalised" (RepetitionPenaltyLogitsProcessor) and
// "banned" (NoRepeatNGramLogitsProcessor's n-gram matches, the eos ids of MinLength / MinNewTokensLength while the
// prefix is shorter than eos_bound), then scores the row in one pass.  Ban and penalty commute (a banned score is
// -inf either way), so the result does not depend on the order HF lists the processors in.
struct ProcessedScore {
  const unsigned* pen;
  const unsigned* ban;
  float pf, inv;
  bool rep;
  __device__ __forceinline__ float operator()(float f, int id) const {
    const unsigned m = 1u << (id & 31);
    const int w = id >> 5;
    // torch on CUDA: `score * penalty` with the penalty cast to fp32, `score / penalty` as score * fp32(1 / penalty)
    if (rep && (pen[w] & m)) f = f < 0.f ? __fmul_rn(f, pf) : __fmul_rn(f, inv);
    return (ban[w] & m) ? -INFINITY : f;
  }
};

template <typename T>
__global__ void __launch_bounds__(256) argmax_processed_kernel(const T* __restrict__ logits, int vocab, int ld,
                                                               const int* __restrict__ st, Dims d,
                                                               const LadeProcessors* __restrict__ proc, int* out_idx) {
  extern __shared__ unsigned s_bits[];          // [words] penalised, then [words] banned
  const int slot = blockIdx.x;
  const int t = threadIdx.x;
  const int flags = proc->flags;
  const int n_out = st[S_N_OUT];
  const int lg = st[S_N_GUESS_TOK];
  int len = -1, g0 = 0;
  if (slot == 0) {
    len = n_out;
  } else if (slot >= 1 + d.WCAP && slot - 1 - d.WCAP < lg) {
    const int i = slot - 1 - d.WCAP;
    const int u = i % d.GS;
    g0 = i - u;
    len = n_out + u + 1;
  }
  if (len < 0 || flags == 0) {
    argmax_row(logits, vocab, ld, slot, IdentityScore(), out_idx);
    return;
  }
  const int words = (vocab + 31) >> 5;
  unsigned* pen = s_bits;
  unsigned* ban = s_bits + words;
  for (int w = t; w < 2 * words; w += blockDim.x) s_bits[w] = 0u;
  __syncthreads();
  const int* out = st + d.off_out;
  const int* gs = st + d.off_guess + g0;
  auto tok = [&](int k) { return k < n_out ? out[k] : gs[k - n_out]; };
  auto mark = [&](unsigned* bits, int id) {
    if (id >= 0 && id < vocab) atomicOr(bits + (id >> 5), 1u << (id & 31));
  };
  const bool rep = (flags & LADE_PROC_REPETITION_PENALTY) != 0;
  if (rep)
    for (int k = max(proc->prompt_ignore_length, 0) + t; k < len; k += blockDim.x) mark(pen, tok(k));
  if (flags & LADE_PROC_NO_REPEAT_NGRAM) {
    // the n-gram starting at j bans its last token when its first n-1 tokens equal the prefix's last n-1
    // (_calc_banned_ngram_tokens; nothing while len + 1 < n, and n = 1 bans every prefix token)
    const int n = proc->ngram_size;
    if (n >= 1 && n <= LADE_PROC_MAX_NGRAM) {
      const int tail = len - n + 1;
      for (int j = t; j <= len - n; j += blockDim.x) {
        bool match = true;
        for (int q = 0; q < n - 1 && match; ++q) match = tok(j + q) == tok(tail + q);
        if (match) mark(ban, tok(j + n - 1));
      }
    }
  }
  if ((flags & LADE_PROC_MIN_LENGTH) && len < proc->eos_bound && t < min(max(proc->n_eos, 0), LADE_PROC_MAX_EOS))
    mark(ban, proc->eos_token_id[t]);
  __syncthreads();
  const float pf = __uint_as_float(proc->penalty_bits);
  ProcessedScore score{pen, ban, pf, __frcp_rn(pf), rep};
  argmax_row(logits, vocab, ld, slot, score, out_idx);
}

// Bitmaps of lade_argmax_processed: two of ceil(vocab / 32) words in dynamic shared memory, kept within the 48 KB a
// launch gets without opting in.
static const int kProcMaxVocab = 160 * 1024;

template <typename T>
static int launch_argmax_processed(LadeCtx* ctx, void* stream, const void* logits, int32_t n_rows, int32_t vocab,
                                   int32_t ld, const LadeProcessors* proc_dev, int32_t* out_idx) {
  if (!ctx || !logits || !proc_dev || !out_idx || n_rows < 1 || vocab < 1 || ld < vocab) return LADE_EINVAL;
  if (vocab > kProcMaxVocab || ctx->d.D != 1) return LADE_EUNSUPPORTED;
  const size_t smem = sizeof(unsigned) * 2 * (size_t)((vocab + 31) / 32);
  argmax_processed_kernel<T><<<n_rows, 256, smem, (cudaStream_t)stream>>>((const T*)logits, vocab, ld, ctx->state,
                                                                          ctx->d, proc_dev, out_idx);
  LADE_LAUNCH_CHECK("argmax_processed_kernel");
  return LADE_OK;
}

static int make_dims(const LadeConfig& c, Dims* d) {
  if (c.level < 3 || c.window_size < 1 || c.vocab_size < 1) return LADE_EINVAL;
  if (c.guess_set_size == -1) return LADE_EUNSUPPORTED;   // unbounded python set (decoding.py:65-78)
  if (c.guess_set_size < 0 || c.max_total_len < 1 || c.n_eos < 0 || c.n_eos > 4) return LADE_EINVAL;
  d->W = c.window_size; d->N = c.level; d->G = c.guess_set_size; d->GS = c.level - 1;
  d->WCAP = c.window_size + c.level - 3;
  d->V = c.vocab_size; d->cap = c.max_total_len; d->pool_from_prompt = c.pool_from_prompt; d->n_eos = c.n_eos;
  for (int i = 0; i < 4; ++i) d->eos[i] = c.eos_token_id[i];
  d->D = c.dist_workers > 1 ? c.dist_workers : 1;
  d->rank = c.dist_workers > 1 ? c.rank : 0;
  if (d->D > 64 || d->rank < 0 || d->rank >= d->D) return LADE_EINVAL;
  // n-gram tuples are staged by one warp, one token per lane: LEVEL - 1 <= 32
  if (d->GS > 32 || d->W > 1024 || d->WCAP > 16384 || d->G > 4096) return LADE_EUNSUPPORTED;
  d->lm_cap = 1 + d->WCAP + d->G * d->GS;
  long long off = S_HDR_INTS;
  d->off_win = (int)off; off += (long long)(d->N - 1) * d->WCAP;
  d->off_win_len = (int)off; off += d->N - 1;
  d->off_guess = (int)off; off += (long long)(d->G > 0 ? d->G : 1) * d->GS;
  d->off_out = (int)off; off += d->cap;
  d->off_old = (int)off; off += d->cap;
  d->off_cnt = (int)off; off += d->V;
  d->off_tup = off; off += (long long)d->V * (d->G > 0 ? d->G : 1) * d->GS;
  d->total_ints = off;
  return LADE_OK;
}

}  // namespace lade

using namespace lade;

extern "C" {

int lade_ctx_create(const LadeConfig* cfg, LadeCtx** out) {
  if (!cfg || !out) return LADE_EINVAL;
  Dims d;
  int rc = make_dims(*cfg, &d);
  if (rc != LADE_OK) return rc;
  LadeCtx* ctx = new (std::nothrow) LadeCtx();
  if (!ctx) return LADE_ENOMEM;
  ctx->cfg = *cfg;
  ctx->d = d;
  ctx->state = nullptr;
  cudaError_t e = cudaMalloc(&ctx->state, sizeof(int32_t) * d.total_ints);
  if (e != cudaSuccess) {
    set_cuda_error(e, "cudaMalloc(state)");
    delete ctx;
    return e == cudaErrorMemoryAllocation ? LADE_ENOMEM : LADE_ECUDA;
  }
  *out = ctx;
  return LADE_OK;
}

int lade_ctx_destroy(LadeCtx* ctx) {
  if (!ctx) return LADE_EINVAL;
  if (ctx->state) cudaFree(ctx->state);
  delete ctx;
  return LADE_OK;
}

int lade_ctx_reset(LadeCtx* ctx, void* stream, const int32_t* prompt_host, int32_t n_prompt,
                   const int32_t* window0_host, int32_t n_window0, int32_t max_length) {
  if (!ctx || !prompt_host || !window0_host) return LADE_EINVAL;
  const Dims& d = ctx->d;
  if (n_prompt < 1 || n_prompt > d.cap || n_window0 != d.WCAP || max_length > d.cap) return LADE_EINVAL;
  cudaStream_t s = (cudaStream_t)stream;
  LADE_CUDA_CHECK(cudaMemsetAsync(ctx->state + d.off_cnt, 0, sizeof(int32_t) * d.V, s));
  LADE_CUDA_CHECK(cudaMemcpyAsync(ctx->state + d.off_out, prompt_host, sizeof(int32_t) * n_prompt,
                                  cudaMemcpyHostToDevice, s));
  LADE_CUDA_CHECK(cudaMemcpyAsync(ctx->state + d.off_win, window0_host, sizeof(int32_t) * n_window0,
                                  cudaMemcpyHostToDevice, s));
  reset_header_kernel<<<1, 256, 0, s>>>(ctx->state, d, n_prompt, n_window0, max_length);
  LADE_LAUNCH_CHECK("reset_header_kernel");
  if (d.pool_from_prompt && d.G > 0) {
    fill_pool_from_prompt_kernel<<<37, 256, 0, s>>>(ctx->state, d, n_prompt);   // 296 warps, keys sharded by id
    LADE_LAUNCH_CHECK("fill_pool_from_prompt_kernel");
  }
  return LADE_OK;
}

int lade_step_layout(LadeCtx* ctx, void* stream, int32_t q_pad, int32_t* ids_out, int32_t* pos_out,
                     int32_t* rowdesc_out, int32_t* lm_rows_out, int32_t* meta_out, uint32_t* rowmask_out,
                     int32_t mask_words) {
  if (!ctx || !ids_out || !pos_out || !rowdesc_out || !lm_rows_out || !meta_out || q_pad < 1) return LADE_EINVAL;
  if (rowmask_out && mask_words * 32 < q_pad && mask_words > 0) return LADE_EINVAL;
  if (ctx->d.N - 1 > 64) return LADE_EUNSUPPORTED;
  step_layout_kernel<<<1, 256, 0, (cudaStream_t)stream>>>(ctx->state, ctx->d, q_pad, ids_out, pos_out,
                                                          rowdesc_out, lm_rows_out, meta_out,
                                                          mask_words > 0 ? rowmask_out : nullptr, mask_words);
  LADE_LAUNCH_CHECK("step_layout_kernel");
  return LADE_OK;
}

int lade_step_rows_bound(const LadeConfig* cfg, int32_t n_prompt, int32_t step_index) {
  if (!cfg || cfg->level < 3 || step_index < 0) return LADE_EINVAL;
  const int W = cfg->window_size, N = cfg->level, G = cfg->guess_set_size > 0 ? cfg->guess_set_size : 0;
  const int D = cfg->dist_workers > 1 ? cfg->dist_workers : 1;
  const int rank = D > 1 ? cfg->rank : 0;
  // level sizes before step k: |L0| = W+N-3-k (k <= N-2), afterwards W-1 ; window_len = |L0|+1
  const int k = step_index < N - 2 ? step_index : N - 2;
  const int len0 = W + N - 3 - k;
  const int window_len = len0 + 1;
  const int split = (window_len + D - 1) / D;
  const int ws = D > 1 ? (split * rank < window_len ? split * rank : window_len) : 0;
  const int we = D > 1 ? (split * (rank + 1) < window_len ? split * (rank + 1) : window_len) : window_len;
  const int l0_in = we - 1 > 0 ? we - 1 : 0;
  const int slice = D > 1 ? we - ws : window_len;   // single GPU: |L_l| = |L0|+1 for l >= 1
  if (step_index == 0) return n_prompt + l0_in;
  if (step_index <= N - 3) return 1 + l0_in + step_index * slice;
  const int skip_max = D > 1 ? N - 2 : 0;            // re-fed accepted tokens (decoding.py:1150)
  const int g_max = (G + D - 1) / D;
  return 1 + skip_max + l0_in + (N - 2) * slice + g_max * (N - 1);
}

int lade_accept_update(LadeCtx* ctx, void* stream, const int32_t* argmax_slots, const int32_t* meta,
                       int32_t* result) {
  if (!ctx || !argmax_slots || !meta || !result) return LADE_EINVAL;
  accept_update_kernel<<<1, 128, 0, (cudaStream_t)stream>>>(ctx->state, ctx->d, argmax_slots, meta, result);
  LADE_LAUNCH_CHECK("accept_update_kernel");
  return LADE_OK;
}

int lade_kv_compact(void* stream, const int32_t* result, void* k_base, void* v_base,
                    int64_t layer_stride_elems, int32_t n_layers, int32_t n_kv_heads,
                    int32_t kv_capacity, int32_t head_dim, int32_t max_rows) {
  if (!result || !k_base || !v_base || n_layers < 1 || head_dim % 8 != 0 || head_dim > 1024 * 8) return LADE_EINVAL;
  if (max_rows < 1) return LADE_OK;
  dim3 grid(n_layers * 2 * n_kv_heads, max_rows);
  int threads = ((head_dim / 8 + 31) / 32) * 32;
  kv_compact_kernel<<<grid, threads, 0, (cudaStream_t)stream>>>(result, (__nv_bfloat16*)k_base,
                                                                (__nv_bfloat16*)v_base, layer_stride_elems,
                                                                n_kv_heads, kv_capacity, head_dim);
  LADE_LAUNCH_CHECK("kv_compact_kernel");
  return LADE_OK;
}

int lade_argmax_rows(void* stream, const void* logits, int32_t n_rows, int32_t vocab, int32_t ld,
                     int32_t* out_idx) {
  if (!logits || !out_idx || n_rows < 1 || vocab < 1 || ld < vocab) return LADE_EINVAL;
  argmax_rows_kernel<__nv_bfloat16><<<n_rows, 256, 0, (cudaStream_t)stream>>>((const __nv_bfloat16*)logits, vocab, ld, out_idx);
  LADE_LAUNCH_CHECK("argmax_rows_kernel");
  return LADE_OK;
}

int lade_argmax_rows_f16(void* stream, const void* logits, int32_t n_rows, int32_t vocab, int32_t ld,
                         int32_t* out_idx) {
  if (!logits || !out_idx || n_rows < 1 || vocab < 1 || ld < vocab) return LADE_EINVAL;
  argmax_rows_kernel<__half><<<n_rows, 256, 0, (cudaStream_t)stream>>>((const __half*)logits, vocab, ld, out_idx);
  LADE_LAUNCH_CHECK("argmax_rows_kernel");
  return LADE_OK;
}

int lade_argmax_processed(LadeCtx* ctx, void* stream, const void* logits, int32_t n_rows, int32_t vocab, int32_t ld,
                          const LadeProcessors* proc_dev, int32_t* out_idx) {
  return launch_argmax_processed<__nv_bfloat16>(ctx, stream, logits, n_rows, vocab, ld, proc_dev, out_idx);
}

int lade_argmax_processed_f16(LadeCtx* ctx, void* stream, const void* logits, int32_t n_rows, int32_t vocab,
                              int32_t ld, const LadeProcessors* proc_dev, int32_t* out_idx) {
  return launch_argmax_processed<__half>(ctx, stream, logits, n_rows, vocab, ld, proc_dev, out_idx);
}

int lade_processors_upload(void* stream, const LadeProcessors* host, LadeProcessors* dev) {
  if (!host || !dev) return LADE_EINVAL;
  const int known = LADE_PROC_REPETITION_PENALTY | LADE_PROC_NO_REPEAT_NGRAM | LADE_PROC_MIN_LENGTH;
  if (host->flags & ~known) return LADE_EINVAL;
  if (host->flags & LADE_PROC_REPETITION_PENALTY) {
    uint32_t b = host->penalty_bits;
    float pf;
    memcpy(&pf, &b, sizeof(pf));
    if (!(pf > 0.f) || !(pf < INFINITY) || host->prompt_ignore_length < 0) return LADE_EINVAL;
  }
  if ((host->flags & LADE_PROC_NO_REPEAT_NGRAM) && (host->ngram_size < 1 || host->ngram_size > LADE_PROC_MAX_NGRAM))
    return LADE_EINVAL;
  if (host->n_eos < 0 || host->n_eos > LADE_PROC_MAX_EOS) return LADE_EINVAL;
  LADE_CUDA_CHECK(cudaMemcpyAsync(dev, host, sizeof(LadeProcessors), cudaMemcpyHostToDevice, (cudaStream_t)stream));
  return LADE_OK;
}

int lade_ctx_output_ids(LadeCtx* ctx, void* stream, int32_t* out_host, int32_t n) {
  if (!ctx || !out_host || n < 0 || n > ctx->d.cap) return LADE_EINVAL;
  LADE_CUDA_CHECK(cudaMemcpyAsync(out_host, ctx->state + ctx->d.off_out, sizeof(int32_t) * n,
                                  cudaMemcpyDeviceToHost, (cudaStream_t)stream));
  LADE_CUDA_CHECK(cudaStreamSynchronize((cudaStream_t)stream));
  return LADE_OK;
}

int lade_ctx_pool_snapshot(LadeCtx* ctx, void* stream, int32_t* cnt_host, int32_t* tup_host) {
  if (!ctx || !cnt_host || !tup_host) return LADE_EINVAL;
  const Dims& d = ctx->d;
  LADE_CUDA_CHECK(cudaMemcpyAsync(cnt_host, ctx->state + d.off_cnt, sizeof(int32_t) * d.V,
                                  cudaMemcpyDeviceToHost, (cudaStream_t)stream));
  LADE_CUDA_CHECK(cudaMemcpyAsync(tup_host, ctx->state + d.off_tup, sizeof(int32_t) * (size_t)d.V * d.G * d.GS,
                                  cudaMemcpyDeviceToHost, (cudaStream_t)stream));
  LADE_CUDA_CHECK(cudaStreamSynchronize((cudaStream_t)stream));
  return LADE_OK;
}

int lade_ctx_window_snapshot(LadeCtx* ctx, void* stream, int32_t* win_host, int32_t* len_host) {
  if (!ctx || !win_host || !len_host) return LADE_EINVAL;
  const Dims& d = ctx->d;
  LADE_CUDA_CHECK(cudaMemcpyAsync(win_host, ctx->state + d.off_win, sizeof(int32_t) * (d.N - 1) * d.WCAP,
                                  cudaMemcpyDeviceToHost, (cudaStream_t)stream));
  LADE_CUDA_CHECK(cudaMemcpyAsync(len_host, ctx->state + d.off_win_len, sizeof(int32_t) * (d.N - 1),
                                  cudaMemcpyDeviceToHost, (cudaStream_t)stream));
  LADE_CUDA_CHECK(cudaStreamSynchronize((cudaStream_t)stream));
  return LADE_OK;
}

int lade_lp_record_ints(const LadeConfig* cfg) {
  if (!cfg || cfg->level < 3) return LADE_EINVAL;
  return 3 + (cfg->level - 1) + (cfg->window_size + cfg->level - 3);
}

int lade_commit_decision(LadeCtx* ctx, void* stream, const int32_t* decision, const int32_t* meta, int32_t* result) {
  if (!ctx || !decision || !meta || !result) return LADE_EINVAL;
  if (ctx->d.D != 1) return LADE_ESTATE;   // the sampling path has no LP (reference: replicas only)
  commit_decision_kernel<<<1, 128, 0, (cudaStream_t)stream>>>(ctx->state, ctx->d, decision, meta, result);
  LADE_LAUNCH_CHECK("commit_decision_kernel");
  return LADE_OK;
}

int lade_lp_verify(LadeCtx* ctx, void* stream, const int32_t* argmax_slots, const int32_t* meta, int32_t* record_out) {
  if (!ctx || !argmax_slots || !meta || !record_out) return LADE_EINVAL;
  lp_verify_kernel<<<1, 128, 0, (cudaStream_t)stream>>>(ctx->state, ctx->d, argmax_slots, meta, record_out);
  LADE_LAUNCH_CHECK("lp_verify_kernel");
  return LADE_OK;
}

int lade_lp_commit(LadeCtx* ctx, void* stream, const int32_t* records_all, const int32_t* meta, int32_t* result) {
  if (!ctx || !records_all || !meta || !result) return LADE_EINVAL;
  lp_commit_kernel<<<1, 128, 0, (cudaStream_t)stream>>>(ctx->state, ctx->d, records_all, meta, result);
  LADE_LAUNCH_CHECK("lp_commit_kernel");
  return LADE_OK;
}

const char* lade_strerror(int code) {
  switch (code) {
    case LADE_OK: return "ok";
    case LADE_EINVAL: return "invalid argument or unsupported shape";
    case LADE_ECUDA: return "CUDA runtime error (see lade_last_cuda_error)";
    case LADE_ENOMEM: return "out of memory";
    case LADE_EUNSUPPORTED: return "unsupported configuration";
    case LADE_ESTATE: return "invalid call sequence";
    default: return "unknown error";
  }
}

const char* lade_last_cuda_error(void) { return lade::g_last_error.c_str(); }

int lade_version(void) { return 103; }

}  // extern "C"
