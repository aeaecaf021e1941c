// ctc_q.cuh -- the CTC arithmetic shared by the lexicon decoder (ctc_lexicon.cu) and the training loss (ctc_train.cu),
// so that both score a text on exactly the same numbers:
//   q[t,c] = softmax(l_t)_c + 1e-7 (= exp(lp[t,c]) of the beam decoder), formed by ctc_step_norm + ctc_q;
//   the states of a label sequence l_1..l_L are ext = (blank, l_1, blank, ..., l_L, blank), S = 2L+1;
//   ctc_need_steps / ctc_prune zero the states that can no longer reach a final state, ctc_rescale keeps the largest
//   state in [2^32, 2^100) by exact powers of two (ctc_lexicon.cu's header gives the argument).
#pragma once
#include <math.h>

namespace ctcq {

constexpr int kT = 48;                                           // kept steps (rnn_steps_to_discard = 2 of 50)

// Max and sum of exp(l - max) of one step's K logits, by one warp (lane l reads classes l, l+32, ...) in a fixed order:
// every lane of the warp returns the same two values.
__device__ __forceinline__ void ctc_step_norm(const float* __restrict__ row, int K, int lane, float* m_out, float* se_out) {
  float m = -INFINITY;
  for (int c = lane; c < K; c += 32) m = fmaxf(m, row[c]);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
  float se = 0.f;
  for (int c = lane; c < K; c += 32) se = __fadd_rn(se, expf(__fsub_rn(row[c], m)));
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) se = __fadd_rn(se, __shfl_xor_sync(0xffffffffu, se, o));
  *m_out = m;
  *se_out = se;
}

// softmax(l)_c of a logit l against its step's (m, se), and q = that + 1e-7.
__device__ __forceinline__ float ctc_p(float l, float m, float se) { return __fdiv_rn(expf(__fsub_rn(l, m)), se); }
__device__ __forceinline__ float ctc_q(float l, float m, float se) { return __fadd_rn(ctc_p(l, m, se), 1e-7f); }

// Multiplies the states by an exact power of two (kept in e_sum) when the largest leaves [2^32, 2^100).
template <int NS>
__device__ __forceinline__ void ctc_rescale(float (&a)[NS], int& e_sum) {
  float m = a[0];
#pragma unroll
  for (int s = 1; s < NS; ++s) m = fmaxf(m, a[s]);
  if (m > 0.f && (m < 0x1p32f || m >= 0x1p100f)) {
    int sh = 99 - ((__float_as_int(m) >> 23) - 127);            // the largest state into [2^99, 2^100)
    sh = max(-126, min(126, sh));
    const float f = __int_as_float((127 + sh) << 23);
#pragma unroll
    for (int s = 0; s < NS; ++s) a[s] = __fmul_rn(a[s], f);
    e_sum += sh;
  }
}

// The shift ctc_rescale applies for a largest state m (0: none), for code that keeps its states outside registers.
__device__ __forceinline__ int ctc_rescale_shift(float m) {
  if (!(m > 0.f) || (m >= 0x1p32f && m < 0x1p100f)) return 0;
  const int sh = 99 - ((__float_as_int(m) >> 23) - 127);
  return max(-126, min(126, sh));
}

// Steps an alignment needs from state s to a final state (S-2 or S-1): one per label still to come, one per blank a
// repeated label among them needs, one more from a blank state.  rep: bit i (0 < i < L) set where label i repeats
// label i-1.
__device__ __forceinline__ int ctc_need_steps(int s, int L, unsigned long long rep) {
  if (s >= 2 * L - 1) return 0;
  const int i = s >> 1;
  return (L - 1 - i) + __popcll(rep >> (i + 1)) + ((s & 1) ? 0 : 1);
}

// Zeroes the states that can no longer reach a final state in the `left` steps that remain.  They are a prefix
// (need_steps does not increase with s), [0, live), and never flow into a state that can: s -> s' in one step means
// need(s) <= need(s') + 1.  So zeroing them changes no score, and the rescaling follows the largest state that counts
// -- without it, a state that stays on blank would hold the scale while the only path to the end underflows.
template <int NS>
__device__ __forceinline__ void ctc_prune(float (&a)[NS], int& live, int left, int L, unsigned long long rep) {
  while (live < 2 * L - 1 && ctc_need_steps(live, L, rep) > left) ++live;
#pragma unroll
  for (int s = 0; s < NS; ++s)
    if (s < live) a[s] = 0.f;
}

}  // namespace ctcq
