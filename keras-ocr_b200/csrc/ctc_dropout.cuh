// ctc_dropout.cuh -- the Dropout(rate) mask on the BiLSTM output that feeds fc_12 (recognition.py:321), shared by the
// output-layer training (ctc_train.cu) and the recurrent-layer training (rnn_train.cu), so both key it the same way:
// feature c of kept step t of dataset row r is kept iff  mix64(key0 ^ (r * 12288 + t * 256 + c)) >> 40  >=  thr =
// floor(rate * 2^24), key0 = mix64(mix64(seed) ^ step), mix64 the splitmix64 finaliser.  A kept feature is multiplied by
// scale = fp32(1 / (1 - rate)), a dropped one is 0; rate 0 leaves the features as they are.
#pragma once

#include <stdint.h>

#include "ctc_q.cuh"

namespace ctcdrop {

constexpr int kFeat = 256;

__host__ __device__ __forceinline__ uint64_t mix64(uint64_t z) {
  z += 0x9E3779B97F4A7C15ull;
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  return z ^ (z >> 31);
}

struct Dropout {
  uint64_t key0;
  unsigned thr;       // keep iff hash >> 40 >= thr
  float scale;
  bool on;
};

inline Dropout make_dropout(float rate, uint64_t seed, uint64_t step) {
  Dropout d;
  d.on = rate > 0.f;
  d.key0 = mix64(mix64(seed) ^ step);
  d.thr = static_cast<unsigned>(static_cast<double>(rate) * 16777216.0);
  d.scale = 1.0f / (1.0f - rate);
  return d;
}

__device__ __forceinline__ bool kept(const Dropout& d, int row, int t, int c) {
  const uint64_t k = static_cast<uint64_t>(row) * (ctcq::kT * kFeat) + static_cast<uint64_t>(t * kFeat + c);
  return static_cast<unsigned>(mix64(d.key0 ^ k) >> 40) >= d.thr;
}

}  // namespace ctcdrop
