// Sampling verification on the device: the multi-candidate rejection test of the sampling lookahead loop
// (lade/decoding.py:445-546, "modified SpecInfer"), for the reference's warper set {temperature, top-k, top-p}
// (decoding.py:375-377).
//
// Reference, per step (host python + eager torch, one .item() sync per candidate, decoding.py:506):
//   probs_next = softmax(out_logits / T)                                              :445,:485
//   for position i of the n-grams:                                                    :491
//     for every n-gram still alive, in pool order:                                    :495
//       accept its token t with probability min(1, probs_next[t])   (random.random()) :505-508
//       on accept: keep only the n-grams that agree on t, continue with probs_next = softmax(guess_logits[row] / T)   :512-530
//       on reject: probs_next[t] = 0 ; probs_next /= probs_next.sum()                 :518-520
//     nobody accepted: emit one token drawn from the residual distribution, stop      :533-535
//   steps without candidates: one multinomial draw from softmax(out_logits / T)       :458-480,:543-546
//   EOS in the newest window row is replaced by a random earlier token                :131-135,:578-580
//
// Here: ONE kernel, one CTA.  Row statistics (max, sum of exp) and the inverse-CDF draw are block-wide passes over the
// vocabulary; the accept chain itself is a handful of scalar steps on thread 0.  Random numbers come from one
// Philox4x32-10 stream (seed, offset) kept in device memory and advanced by the kernel, so the step -- forward, this
// kernel, lade_commit_decision, KV compaction -- replays from one CUDA graph with no host round trip.  Renormalising
// after k rejections is carried as the rejected mass: p'[t] = p[t] / (1 - sum of rejected p) (exactly what the
// sequential divide-by-sum computes, without rewriting 32000 probabilities per rejection).
#include "state.cuh"

#include <curand_kernel.h>

namespace lade {

constexpr int SMP_THREADS = 1024;
constexpr int SMP_MAX_NGRAMS = 1024;

__device__ __forceinline__ float block_reduce_max(float v, float* s_red) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  __syncthreads();
  if (lane == 0) s_red[warp] = v;
  __syncthreads();
  float r = (lane < (int)(blockDim.x >> 5)) ? s_red[lane] : -INFINITY;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) r = fmaxf(r, __shfl_xor_sync(0xffffffffu, r, o));
  return r;      // every thread holds the block maximum
}

__device__ __forceinline__ float block_reduce_sum(float v, float* s_red) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  __syncthreads();
  if (lane == 0) s_red[warp] = v;
  __syncthreads();
  float r = (lane < (int)(blockDim.x >> 5)) ? s_red[lane] : 0.f;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) r += __shfl_xor_sync(0xffffffffu, r, o);
  return r;
}

// scores = logits / T in fp32 (TemperatureLogitsWarper), softmax in fp32
template <typename T>
__device__ __forceinline__ float score_of(const T* row, int t, float temperature) {
  return Elem<T>::to_f(row[t]) / temperature;
}

// 16-bit float bit pattern (bf16 or fp16: sign-magnitude) -> 16-bit key that orders like the value (the logits have a
// 16-bit dtype: at most 65536 distinct scores, so top-k / top-p cut-offs are exact thresholds on this key, found with
// two 256-bin histograms instead of a sort)
template <typename T>
__device__ __forceinline__ unsigned key_of(T x) {
  unsigned b = Elem<T>::key16(x);
  if (b == 0x8000u) b = 0u;          // -0 and +0 are one value to the warpers' comparisons: one key
  return (b & 0x8000u) ? (~b & 0xffffu) : (b | 0x8000u);
}

// The warped distribution of one logits row: p[t] = (key(t) >= thr) * exp(score_t - mx) / sum.
struct RowDist { float mx, sum; unsigned thr; };

template <typename T>
__device__ __forceinline__ float e_of(const T* row, int t, float temperature, const RowDist& d) {
  return key_of(row[t]) >= d.thr ? __expf(score_of(row, t, temperature) - d.mx) : 0.f;
}

// TemperatureLogitsWarper -> TopKLogitsWarper (keep every score >= the k-th largest, ties included) ->
// TopPLogitsWarper (ascending cumulative probability of the top-k-filtered softmax: drop while cum <= 1 - top_p;
// min_tokens_to_keep = 1).  Scores tie in whole buckets of equal bf16 value; a bucket is dropped only when all of it
// can go (torch.sort breaks such ties arbitrarily, so there is no reference order to follow inside a bucket).
template <typename T>
__device__ RowDist row_dist(const T* row, int vocab, float temperature, int top_k, float top_p, float* s_red,
                            int* s_cnt, unsigned long long* s_mass, unsigned long long* s_mtot, int* s_sel) {
  RowDist d;
  float mx = -INFINITY;
  unsigned kmax = 0;
  for (int t = threadIdx.x; t < vocab; t += blockDim.x) {
    mx = fmaxf(mx, score_of(row, t, temperature));
    kmax = max(kmax, key_of(row[t]));
  }
  d.mx = block_reduce_max(mx, s_red);
  const unsigned top_key = (unsigned)block_reduce_max((float)kmax, s_red);        // 16-bit keys are exact in fp32
  d.thr = 0;
  if (top_k > 0 && top_k < vocab) {
    for (int pass = 0; pass < 2; ++pass) {                   // pass 0: high byte, pass 1: low byte inside that bucket
      for (int i = threadIdx.x; i < 256; i += blockDim.x) s_cnt[i] = 0;
      __syncthreads();
      const unsigned hb = pass ? (unsigned)s_sel[0] : 0u;
      for (int t = threadIdx.x; t < vocab; t += blockDim.x) {
        const unsigned k = key_of(row[t]);
        if (pass == 0) atomicAdd(&s_cnt[k >> 8], 1);
        else if ((k >> 8) == hb) atomicAdd(&s_cnt[k & 255u], 1);
      }
      __syncthreads();
      if (threadIdx.x == 0) {
        int cum = pass ? s_sel[1] : 0;                       // elements in strictly higher buckets
        int b = 255;
        for (; b > 0; --b) {
          if (cum + s_cnt[b] >= top_k) break;
          cum += s_cnt[b];
        }
        if (pass == 0) { s_sel[0] = b; s_sel[1] = cum; }
        else s_sel[2] = b;
      }
      __syncthreads();
    }
    d.thr = ((unsigned)s_sel[0] << 8) | (unsigned)s_sel[2];
    __syncthreads();
  }
  float sm = 0.f;
  for (int t = threadIdx.x; t < vocab; t += blockDim.x)
    if (key_of(row[t]) >= d.thr) sm += __expf(score_of(row, t, temperature) - d.mx);
  d.sum = block_reduce_sum(sm, s_red);
  if (top_p < 1.f) {
    // Bucket masses in 2^-40 fixed point (every e <= 1, so even 2^17 terms stay below 2^57).  Integer adds are exact:
    // the cut does not depend on the order of the atomics, and the kept mass total - dropped has no cancellation.
    for (int pass = 0; pass < 2; ++pass) {
      for (int i = threadIdx.x; i < 256; i += blockDim.x) s_mass[i] = 0ull;
      __syncthreads();
      const unsigned hb = pass ? (unsigned)s_sel[0] : 0u;
      for (int t = threadIdx.x; t < vocab; t += blockDim.x) {
        const unsigned k = key_of(row[t]);
        if (k < d.thr) continue;
        const unsigned long long e = __float2ull_rn(__expf(score_of(row, t, temperature) - d.mx) * 0x1p40f);
        if (pass == 0) atomicAdd(&s_mass[k >> 8], e);
        else if ((k >> 8) == hb) atomicAdd(&s_mass[k & 255u], e);
      }
      __syncthreads();
      if (threadIdx.x == 0) {
        if (pass == 0) {
          unsigned long long total = 0;
          for (int b = 0; b < 256; ++b) total += s_mass[b];
          s_mtot[0] = total;
          s_mtot[1] = 0;                                     // mass of the buckets already dropped
        }
        const double lim = (1.0 - (double)top_p) * (double)s_mtot[0];
        unsigned long long cum = s_mtot[1];
        // min_tokens_to_keep = 1: the scan stops at the bucket of the largest key at the latest
        const int last = pass ? ((top_key >> 8) == hb ? (int)(top_key & 255u) : 255) : (int)(top_key >> 8);
        int b = 0;
        for (; b < last; ++b) {
          if (!((double)(cum + s_mass[b]) <= lim)) break;    // this bucket crosses 1 - top_p: it stays
          cum += s_mass[b];
        }
        if (pass == 0) s_sel[0] = b;
        else s_sel[2] = b;
        s_mtot[1] = cum;
      }
      __syncthreads();
    }
    const unsigned thr_p = ((unsigned)s_sel[0] << 8) | (unsigned)s_sel[2];
    const unsigned long long kept = s_mtot[0] - s_mtot[1];
    __syncthreads();
    if (thr_p > d.thr) { d.thr = thr_p; d.sum = (float)((double)kept * 0x1p-40); }
  }
  if (d.thr > top_key) d.thr = top_key;
  return d;
}

// Cut-offs of the three threshold warpers after top-p (0 = off; the C-ABI has checked the ranges).
struct Warpers { float min_p, epsilon, eta; };

// Smallest key among the kept tokens (key >= thr) that pass `keep`; thr itself when none does.  Every warper below
// keeps the top token, so the result never exceeds the top key.
template <typename T, typename Keep>
__device__ __forceinline__ unsigned min_kept_key(const T* row, int vocab, unsigned thr, Keep keep, float* s_red) {
  float best = -65536.f;                                     // max of -key: 16-bit keys are exact in fp32
  for (int t = threadIdx.x; t < vocab; t += blockDim.x) {
    const unsigned k = key_of(row[t]);
    if (k >= thr && keep(t)) best = fmaxf(best, -(float)k);
  }
  const float r = -block_reduce_max(best, s_red);
  return r > 65535.f ? thr : (unsigned)r;
}

// (S, sum of e_t x_t) over the kept tokens, x_t = score_t - mx, e_t = exp(x_t): the mass and the entropy term.
template <typename T>
__device__ __forceinline__ float2 kept_moments(const T* row, int vocab, float temperature, const RowDist& d,
                                               float* s_red) {
  float sm = 0.f, sx = 0.f;
  for (int t = threadIdx.x; t < vocab; t += blockDim.x) {
    if (key_of(row[t]) < d.thr) continue;
    const float x = score_of(row, t, temperature) - d.mx;
    const float e = __expf(x);
    sm += e;
    if (e > 0.f) sx += e * x;                                // an underflowed term adds nothing (and no -inf * 0)
  }
  return make_float2(block_reduce_sum(sm, s_red), block_reduce_sum(sx, s_red));
}

// row_dist followed by MinPLogitsWarper -> EpsilonLogitsWarper -> EtaLogitsWarper (HF's list order; each acts on the
// softmax of what the previous ones kept; min_tokens_to_keep = 1, filter value -inf).  With p_t = e_t / S:
// * MinP drops p_t < min_p * max p, i.e. e_t < min_p (the top token's e is 1);
// * Epsilon drops p_t < epsilon unless the score is the maximum;
// * Eta drops p_t < min(eta, sqrt(eta) exp(-H)), H = ln S - sum(e_t x_t) / S the entropy of the kept distribution,
//   again unless the score is the maximum.
// A cut is a threshold on the key (the score is monotone in it), so each is one more pass for the smallest key that
// stays, and the kept set stays an upper set of the key.  d.sum is recomputed over the final kept set whenever a cut
// moved the threshold (the top-p kept mass no longer applies then).  `wdbg` (nullable): per visited row, the final
// threshold key and S'.
template <typename T>
__device__ RowDist row_dist_warped(const T* row, int vocab, float temperature, int top_k, float top_p, const Warpers& w,
                                   float* s_red, int* s_cnt, unsigned long long* s_mass, unsigned long long* s_mtot,
                                   int* s_sel, float* wdbg) {
  RowDist d = row_dist(row, vocab, temperature, top_k, top_p, s_red, s_cnt, s_mass, s_mtot, s_sel);
  bool stale = false;                                        // d.sum is not the mass of the current kept set
  if (w.min_p > 0.f) {
    const float mp = w.min_p;
    const unsigned thr = min_kept_key(row, vocab, d.thr, [&](int t) {
      return __expf(score_of(row, t, temperature) - d.mx) >= mp; }, s_red);
    if (thr > d.thr) { d.thr = thr; stale = true; }
  }
  if (w.epsilon > 0.f) {
    if (stale) { d.sum = kept_moments(row, vocab, temperature, d, s_red).x; stale = false; }
    const float eps = w.epsilon, S = d.sum;
    const unsigned thr = min_kept_key(row, vocab, d.thr, [&](int t) {
      const float s = score_of(row, t, temperature);
      return s == d.mx || !(__expf(s - d.mx) / S < eps); }, s_red);
    if (thr > d.thr) { d.thr = thr; stale = true; }
  }
  if (w.eta > 0.f) {
    const float2 m = kept_moments(row, vocab, temperature, d, s_red);
    d.sum = m.x;
    stale = false;
    const float ent = logf(m.x) - m.y / m.x;
    const float eta = fminf(w.eta, sqrtf(w.eta) * expf(-ent)), S = d.sum;
    const unsigned thr = min_kept_key(row, vocab, d.thr, [&](int t) {
      const float s = score_of(row, t, temperature);
      return s == d.mx || !(__expf(s - d.mx) / S < eta); }, s_red);
    if (thr > d.thr) { d.thr = thr; stale = true; }
  }
  if (stale) d.sum = kept_moments(row, vocab, temperature, d, s_red).x;
  if (wdbg && threadIdx.x == 0) {
    const int n = (int)wdbg[0];
    wdbg[1 + 2 * n] = (float)d.thr;
    wdbg[2 + 2 * n] = d.sum;
    wdbg[0] = (float)(n + 1);
  }
  return d;
}

// One draw from the distribution e_t = exp(score_t - mx) over t not in zset[0..n_z), by inverse CDF:
// the smallest t whose running mass reaches u * total.  Each thread owns one contiguous chunk of the vocabulary.
template <typename T>
__device__ int multinomial_excluding(const T* row, int vocab, float temperature, const RowDist& rd, float u,
                                     const int* zset, int n_z, float* s_scan, int* s_pick) {
  const int chunk = (vocab + blockDim.x - 1) / blockDim.x;
  const int lo = threadIdx.x * chunk, hi = min(vocab, lo + chunk);
  float local = 0.f;
  for (int t = lo; t < hi; ++t) {
    bool z = false;
    for (int k = 0; k < n_z; ++k) z = z || (zset[k] == t);
    if (!z) local += e_of(row, t, temperature, rd);
  }
  __syncthreads();
  s_scan[threadIdx.x] = local;
  if (threadIdx.x == 0) *s_pick = -1;
  __syncthreads();
  // inclusive scan of the per-thread masses (Hillis-Steele over <= 1024 entries)
  for (int o = 1; o < (int)blockDim.x; o <<= 1) {
    const float add = threadIdx.x >= o ? s_scan[threadIdx.x - o] : 0.f;
    __syncthreads();
    s_scan[threadIdx.x] += add;
    __syncthreads();
  }
  const float total = s_scan[blockDim.x - 1];
  const float target = u * total;
  const float before = threadIdx.x ? s_scan[threadIdx.x - 1] : 0.f;
  const float upto = s_scan[threadIdx.x];
  if (local > 0.f && target > before && target <= upto) {
    float run = before;
    int pick = -1;
    for (int t = lo; t < hi; ++t) {
      bool z = false;
      for (int k = 0; k < n_z; ++k) z = z || (zset[k] == t);
      if (z) continue;
      const float e = e_of(row, t, temperature, rd);
      if (e <= 0.f) continue;
      pick = t;                        // last live token of the chunk if rounding leaves `run` just short
      run += e;
      if (run >= target) break;
    }
    atomicMax(s_pick, pick);           // adjacent chunks can both claim an exact boundary: take one deterministically
  }
  __syncthreads();
  int pick = *s_pick;
  if (pick < 0) {                      // u * total rounded past every chunk: the last token with mass
    if (threadIdx.x == 0) {
      for (int t = vocab - 1; t >= 0 && pick < 0; --t) {
        bool z = false;
        for (int k = 0; k < n_z; ++k) z = z || (zset[k] == t);
        if (!z && e_of(row, t, temperature, rd) > 0.f) pick = t;
      }
      *s_pick = pick < 0 ? 0 : pick;
    }
    __syncthreads();
    pick = *s_pick;
  }
  __syncthreads();
  return pick;
}

// decision_out: the record lade_commit_decision consumes --
//   [first hit, max_hit, n_new, hits[GS], new_tok[WCAP] | max_hit_idx, flags (1 sampling, 2 filtered row present),
//    finished-by-extra-eos, 0, filtered[W]]
// The whole verification of one step; WARPED adds the cuts of row_dist_warped to every row the chain visits.
template <typename T, bool WARPED>
__device__ __forceinline__ void sample_verify_chain(int* st, const Dims& d, const T* __restrict__ logits, int ld, int vocab,
                                                    const int* __restrict__ am, const int* __restrict__ meta,
                                                    float temperature, int top_k, float top_p, const Warpers& wp,
                                                    unsigned long long* rng_state, int* __restrict__ rec, float* dbg,
                                                    float* wdbg) {
  __shared__ float s_red[32];
  __shared__ int s_cnt[256];
  __shared__ unsigned long long s_mass[256];
  __shared__ unsigned long long s_mtot[2];
  __shared__ int s_sel[4];
  __shared__ float s_scan[SMP_THREADS];
  __shared__ int s_pick;
  __shared__ int s_z[SMP_MAX_NGRAMS];           // tokens rejected at the current position
  __shared__ unsigned char s_alive[SMP_MAX_NGRAMS];
  __shared__ int s_ctl[8];                      // 0 accepted?, 1 row of the next distribution, 2 n_z, 3 n_hits, 4 max_hit_idx
  __shared__ float s_u;
  __shared__ int s_hits[64];

  const int t = threadIdx.x;
  const int GS = d.GS, WCAP = d.WCAP, W = d.W;
  const int R = lp_rec_ints(d);
  if (st[S_DONE]) {                             // finished sequence: the commit kernel ignores the record
    for (int i = t; i < R + 4 + W; i += blockDim.x) rec[i] = 0;
    return;
  }
  const int phase = meta[LADE_M_PHASE];
  const int tiny = meta[LADE_M_TINY];
  const int lg = meta[LADE_M_N_GUESS_TOK];
  const int n_ng = lg / GS;
  const int* gtok = st + d.off_guess;
  curandStatePhilox4_32_10_t rng;
  unsigned long long n_draws = 0;
  if (t == 0) curand_init(rng_state[0], 0ull, rng_state[1], &rng);
  int n_dbg = 0;
  auto draw = [&]() {                           // thread 0 only; uniform in (0, 1]
    const float u = curand_uniform(&rng);
    ++n_draws;
    if (dbg) dbg[1 + n_dbg++] = u;
    return u;
  };

  const T* row0 = logits;                       // slot 0 = the next-token row (lade_step_layout's lm_rows)
  if (phase != 2 || n_ng == 0) {                // :458-480, :543-546
    RowDist rs;
    if constexpr (WARPED) rs = row_dist_warped(row0, vocab, temperature, top_k, top_p, wp, s_red, s_cnt, s_mass, s_mtot,
                                               s_sel, wdbg);
    else rs = row_dist(row0, vocab, temperature, top_k, top_p, s_red, s_cnt, s_mass, s_mtot, s_sel);
    if (t == 0) s_u = draw();
    __syncthreads();
    const int tok = multinomial_excluding(row0, vocab, temperature, rs, s_u, s_z, 0, s_scan, &s_pick);
    if (t == 0) { s_hits[0] = tok; s_ctl[3] = 1; s_ctl[4] = 0; }
  } else {                                      // :484-540
    for (int e = t; e < n_ng; e += blockDim.x) s_alive[e] = 1;
    if (t == 0) { s_ctl[1] = 0; s_ctl[3] = 0; s_ctl[4] = 0; }
    __syncthreads();
    for (int i = 0; i < GS; ++i) {
      const int cur = s_ctl[1];
      const T* row = logits + (long long)cur * ld;
      RowDist rs;
      if constexpr (WARPED) rs = row_dist_warped(row, vocab, temperature, top_k, top_p, wp, s_red, s_cnt, s_mass, s_mtot,
                                                 s_sel, wdbg);
      else rs = row_dist(row, vocab, temperature, top_k, top_p, s_red, s_cnt, s_mass, s_mtot, s_sel);
      if (t == 0) {
        int n_z = 0;
        float zmass = 0.f;                      // probability mass rejected so far at this position
        int accepted = 0;
        for (int e = 0; e < n_ng && !accepted; ++e) {
          if (!s_alive[e]) continue;
          const int draft = gtok[e * GS + i];
          bool in_z = false;
          for (int k = 0; k < n_z; ++k) in_z = in_z || (s_z[k] == draft);
          const float p_raw = e_of(row, draft, temperature, rs) / rs.sum;
          const float denom = 1.f - zmass;
          const float p = in_z ? 0.f : (denom > 0.f ? p_raw / denom : 1.f);
          const float u = draw();
          if (u < fminf(1.f, p)) {              // :508 (strict <)
            accepted = 1;
            s_hits[i] = draft;
            s_ctl[4] = e;
            for (int e2 = 0; e2 < n_ng; ++e2)   // :513-516 keep the n-grams that agree on this token
              if (s_alive[e2] && gtok[e2 * GS + i] != draft) s_alive[e2] = 0;
            s_ctl[1] = 1 + WCAP + e * GS + i;   // next distribution: the logits row after this guess token
          } else if (!in_z) {                   // :518-520
            s_z[n_z++] = draft;
            zmass += p_raw;
          }
        }
        s_ctl[0] = accepted;
        s_ctl[2] = n_z;
        if (accepted) s_ctl[3] = i + 1;
        else s_u = draw();
      }
      __syncthreads();
      if (!s_ctl[0]) {                          // :533-535 residual draw, stop
        const int tok = multinomial_excluding(row, vocab, temperature, rs, s_u, s_z, s_ctl[2], s_scan, &s_pick);
        if (t == 0) { s_hits[i] = tok; s_ctl[3] = i + 1; }
        __syncthreads();
        break;
      }
      __syncthreads();
    }
  }
  __syncthreads();
  const int n_hits = s_ctl[3];
  const int max_hit = n_hits - 1;
  // ---- record
  for (int i = t; i < R + 4 + W; i += blockDim.x) rec[i] = 0;
  __syncthreads();
  if (t < GS) rec[3 + t] = t < n_hits ? s_hits[t] : 0;
  for (int j = t; j < WCAP; j += blockDim.x) rec[3 + GS + j] = j < tiny ? am[1 + j] : 0;
  if (t == 0) {
    rec[0] = s_hits[0];
    rec[1] = max_hit;
    rec[2] = tiny;
    rec[R] = max_hit > 0 ? s_ctl[4] : 0;
    int flags = 1;
    // EOS in the newest window row -> a random earlier token (filter_window :131-135 through set_token = copy_from
    // :336-351); the pool is fed the unfiltered row (:563 before :578)
    if (phase == 2 && d.n_eos > 0) {
      flags |= 2;
      const int n_old = st[S_N_OLD];
      const int* old = st + d.off_old;
      for (int j = 0; j < W; ++j) {
        int v = am[1 + j];
        if (v == d.eos[0] && n_old > 0) {
          int k = (int)(draw() * (float)n_old);
          if (k >= n_old) k = n_old - 1;
          v = old[k];
        }
        rec[R + 4 + j] = v;
      }
    }
    rec[R + 1] = flags;
    // the reference refreshes `next_tokens` only on the no-candidate branches (:462,:472,:545): there a drawn token
    // that is one of the further eos ids ends the generation (:636-643); eos[0] among the hits is handled by the
    // emission loop of the commit kernel
    int extra = 0;
    if (phase != 2 || n_ng == 0)
      for (int k = 0; k < d.n_eos; ++k) extra = extra || (s_hits[0] == d.eos[k]);
    rec[R + 2] = extra;
    rng_state[1] += (n_draws + 3ull) & ~3ull;   // Philox yields 4 words per counter value
    if (dbg) dbg[0] = (float)n_dbg;
  }
}

template <typename T>
__global__ void __launch_bounds__(SMP_THREADS, 1)
sample_verify_kernel(int* st, Dims d, const T* __restrict__ logits, int ld, int vocab,
                     const int* __restrict__ am, const int* __restrict__ meta, float temperature, int top_k, float top_p,
                     unsigned long long* rng_state, int* __restrict__ rec, float* dbg) {
  sample_verify_chain<T, false>(st, d, logits, ld, vocab, am, meta, temperature, top_k, top_p, Warpers{0.f, 0.f, 0.f},
                                rng_state, rec, dbg, nullptr);
}

// sample_verify_kernel with MinP / Epsilon / Eta after top-p.  wdbg (nullable): [rows visited, (thr, S') per row].
template <typename T>
__global__ void __launch_bounds__(SMP_THREADS, 1)
sample_verify_warped_kernel(int* st, Dims d, const T* __restrict__ logits, int ld, int vocab,
                            const int* __restrict__ am, const int* __restrict__ meta, float temperature, int top_k,
                            float top_p, Warpers wp, unsigned long long* rng_state, int* __restrict__ rec, float* dbg,
                            float* wdbg) {
  if (wdbg && threadIdx.x == 0) wdbg[0] = 0.f;
  sample_verify_chain<T, true>(st, d, logits, ld, vocab, am, meta, temperature, top_k, top_p, wp, rng_state, rec, dbg,
                               wdbg);
}

}  // namespace lade

using namespace lade;

template <typename T>
static int sample_verify_impl(LadeCtx* ctx, void* stream, const void* logits, int32_t ld, int32_t vocab,
                              const int32_t* argmax_slots, const int32_t* meta, float temperature, int32_t top_k, float top_p,
                              uint64_t* rng_state, int32_t* decision_out, float* debug_uniforms) {
  if (!ctx || !logits || !argmax_slots || !meta || !rng_state || !decision_out) return LADE_EINVAL;
  if (!(temperature > 0.f) || vocab < 1 || ld < vocab || top_k < 0 || !(top_p > 0.f) || top_p > 1.f) return LADE_EINVAL;
  if (ctx->d.D != 1) return LADE_ESTATE;                                   // no LP on the sampling path
  if (ctx->d.G > SMP_MAX_NGRAMS || ctx->d.GS > 64) return LADE_EUNSUPPORTED;
  sample_verify_kernel<T><<<1, SMP_THREADS, 0, (cudaStream_t)stream>>>(
      ctx->state, ctx->d, (const T*)logits, ld, vocab, argmax_slots, meta, temperature, top_k, top_p,
      reinterpret_cast<unsigned long long*>(rng_state), decision_out, debug_uniforms);
  LADE_LAUNCH_CHECK("sample_verify_kernel");
  return LADE_OK;
}

// MinP / epsilon / eta ranges of HF's constructors (0 = off); NaN fails every comparison
static bool warpers_valid(const LadeWarpers& w) {
  const bool cut_ok = (w.min_p >= 0.f && w.min_p <= 1.f) && (w.epsilon == 0.f || (w.epsilon > 0.f && w.epsilon < 1.f)) &&
                      (w.eta == 0.f || (w.eta > 0.f && w.eta < 1.f));
  return cut_ok && w.temperature > 0.f && w.top_k >= 0 && w.top_p > 0.f && w.top_p <= 1.f;
}

template <typename T>
static int sample_verify_warped_impl(LadeCtx* ctx, void* stream, const void* logits, int32_t ld, int32_t vocab,
                                     const int32_t* argmax_slots, const int32_t* meta, const LadeWarpers* w,
                                     uint64_t* rng_state, int32_t* decision_out, float* debug_uniforms,
                                     float* debug_cuts) {
  if (!ctx || !logits || !argmax_slots || !meta || !w || !rng_state || !decision_out) return LADE_EINVAL;
  if (!warpers_valid(*w) || vocab < 1 || ld < vocab) return LADE_EINVAL;
  if (ctx->d.D != 1) return LADE_ESTATE;
  if (ctx->d.G > SMP_MAX_NGRAMS || ctx->d.GS > 64) return LADE_EUNSUPPORTED;
  sample_verify_warped_kernel<T><<<1, SMP_THREADS, 0, (cudaStream_t)stream>>>(
      ctx->state, ctx->d, (const T*)logits, ld, vocab, argmax_slots, meta, w->temperature, w->top_k, w->top_p,
      Warpers{w->min_p, w->epsilon, w->eta}, reinterpret_cast<unsigned long long*>(rng_state), decision_out,
      debug_uniforms, debug_cuts);
  LADE_LAUNCH_CHECK("sample_verify_warped_kernel");
  return LADE_OK;
}

extern "C" {

int lade_sample_verify(LadeCtx* ctx, void* stream, const void* logits, int32_t ld, int32_t vocab,
                       const int32_t* argmax_slots, const int32_t* meta, float temperature, int32_t top_k, float top_p,
                       uint64_t* rng_state, int32_t* decision_out, float* debug_uniforms) {
  return sample_verify_impl<__nv_bfloat16>(ctx, stream, logits, ld, vocab, argmax_slots, meta, temperature, top_k, top_p,
                                           rng_state, decision_out, debug_uniforms);
}

int lade_sample_verify_f16(LadeCtx* ctx, void* stream, const void* logits, int32_t ld, int32_t vocab,
                           const int32_t* argmax_slots, const int32_t* meta, float temperature, int32_t top_k, float top_p,
                           uint64_t* rng_state, int32_t* decision_out, float* debug_uniforms) {
  return sample_verify_impl<__half>(ctx, stream, logits, ld, vocab, argmax_slots, meta, temperature, top_k, top_p,
                                    rng_state, decision_out, debug_uniforms);
}

int lade_sample_verify_warped(LadeCtx* ctx, void* stream, const void* logits, int32_t ld, int32_t vocab,
                              const int32_t* argmax_slots, const int32_t* meta, const LadeWarpers* warpers,
                              uint64_t* rng_state, int32_t* decision_out, float* debug_uniforms, float* debug_cuts) {
  return sample_verify_warped_impl<__nv_bfloat16>(ctx, stream, logits, ld, vocab, argmax_slots, meta, warpers, rng_state,
                                                  decision_out, debug_uniforms, debug_cuts);
}

int lade_sample_verify_warped_f16(LadeCtx* ctx, void* stream, const void* logits, int32_t ld, int32_t vocab,
                                  const int32_t* argmax_slots, const int32_t* meta, const LadeWarpers* warpers,
                                  uint64_t* rng_state, int32_t* decision_out, float* debug_uniforms, float* debug_cuts) {
  return sample_verify_warped_impl<__half>(ctx, stream, logits, ld, vocab, argmax_slots, meta, warpers, rng_state,
                                           decision_out, debug_uniforms, debug_cuts);
}

}  // extern "C"
