// Counter-based Philox4x32-10 shared by the CPU and sm_90a samplers.
//
// Every random decision in the engine is a pure function of
//   (seed, stream, row, draw)
// so the CPU reference path and the CUDA kernels draw the *same* samples and a
// (seed, epoch, batch) triple is enough to replay a loader position.  The
// reference seeds cuRAND from a host mt19937 per launch
// (reference: csrc/cuda/random_sampler.cu:236-241), which is neither
// reproducible across devices nor checkpointable.
#pragma once
#include <algorithm>
#include <cstdint>
#include <cmath>

#if defined(__CUDACC__)
#define GLT_HD __host__ __device__ __forceinline__
#else
#define GLT_HD inline
#endif

namespace glt {

struct U4 { uint32_t x, y, z, w; };

GLT_HD uint32_t mulhi32(uint32_t a, uint32_t b) {
#if defined(__CUDA_ARCH__)
  return __umulhi(a, b);
#else
  return static_cast<uint32_t>((static_cast<uint64_t>(a) * b) >> 32);
#endif
}

GLT_HD U4 philox4x32_10(uint32_t k0, uint32_t k1, U4 c) {
  const uint32_t M0 = 0xD2511F53u, M1 = 0xCD9E8D57u;
  const uint32_t W0 = 0x9E3779B9u, W1 = 0xBB67AE85u;
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    uint32_t hi0 = mulhi32(M0, c.x), lo0 = M0 * c.x;
    uint32_t hi1 = mulhi32(M1, c.z), lo1 = M1 * c.z;
    U4 n;
    n.x = hi1 ^ c.y ^ k0;
    n.y = lo1;
    n.z = hi0 ^ c.w ^ k1;
    n.w = lo0;
    c = n;
    k0 += W0;
    k1 += W1;
  }
  return c;
}

// The i-th 32-bit draw of the stream identified by (seed, stream, row).
GLT_HD uint32_t philox_draw(uint64_t seed, uint32_t stream, uint64_t row, uint32_t i) {
  U4 c;
  c.x = static_cast<uint32_t>(row);
  c.y = static_cast<uint32_t>(row >> 32);
  c.z = i >> 2;
  c.w = stream;
  U4 r = philox4x32_10(static_cast<uint32_t>(seed), static_cast<uint32_t>(seed >> 32), c);
  switch (i & 3u) {
    case 0: return r.x;
    case 1: return r.y;
    case 2: return r.z;
    default: return r.w;
  }
}

// Unbiased-enough bounded draw in [0, n) (Lemire multiply-shift, no rejection).
GLT_HD uint32_t bounded(uint32_t r, uint32_t n) { return mulhi32(r, n); }

// 53-bit uniform double / 24-bit uniform float in [0,1).
GLT_HD float u01(uint32_t r) { return (r >> 8) * (1.0f / 16777216.0f); }

// Exponential-race key for weighted sampling without replacement: the k
// smallest keys of a row are a weighted k-sample (Efraimidis-Spirakis).
GLT_HD float weighted_key(uint64_t seed, uint32_t stream, uint64_t row, uint32_t j, float w) {
  float u = ((philox_draw(seed, stream, row, j) >> 8) + 1u) * (1.0f / 16777216.0f);
  return (w > 0.f) ? (-logf(u) / w) : 3.0e38f;
}

// Floyd's k-subset step i (0-based) of a row with degree d > k:
//   j = d - k + i;  t = U[0, j];  pick = (t already chosen) ? j : t
// Caller supplies the membership test; this only produces t.
GLT_HD uint32_t floyd_candidate(uint64_t seed, uint32_t stream, uint64_t row,
                                uint32_t i, uint32_t d, uint32_t k) {
  uint32_t j = d - k + i;
  return bounded(philox_draw(seed, stream, row, i), j + 1u);
}

// node2vec's second-order step, shared by every walk sampler on both planes.  At v with previous node t, entry x of
// v's row weighs 1/p if x == t, 1 if t's row holds x, 1/q otherwise; the step proposes x uniformly over the row's
// positions and accepts it with probability w(x) / max(1, 1/p, 1/q).  With r = max / min weight <= kNode2VecMaxRatio
// a proposal is accepted with probability >= 1/64, so a step that still has none after kNode2VecMaxProposals takes its
// last proposal with probability < (63/64)^4096 ~ 1e-28.
constexpr int kNode2VecMaxProposals = 4096;
constexpr double kNode2VecMaxRatio = 64.0;

// The three weights divided by their maximum, rounded to float once on the host: every plane then decides a proposal
// with the same float comparisons, so GPU and CPU walks agree bit for bit at any p and q.
struct Node2VecWeights {
  float ret, in, out;
  float lo, hi;  // min / max of in and out: a uniform outside [lo, hi) decides x != t without t's row
};

// nullptr with *w filled, or why p and q are refused.
inline const char* node2vec_weights(double p, double q, Node2VecWeights* w) {
  if (!(std::isfinite(p) && std::isfinite(q) && p > 0 && q > 0)) return "p and q must be finite and > 0";
  const double hi = std::max({1.0, 1.0 / p, 1.0 / q}), lo = std::min({1.0, 1.0 / p, 1.0 / q});
  if (hi / lo > kNode2VecMaxRatio) return "max(1, 1/p, 1/q) / min(1, 1/p, 1/q) must be <= 64";
  w->ret = static_cast<float>(1.0 / p / hi);
  w->in = static_cast<float>(1.0 / hi);
  w->out = static_cast<float>(1.0 / q / hi);
  w->lo = std::min(w->in, w->out);
  w->hi = std::max(w->in, w->out);
  return nullptr;
}

// Accept proposal x, u = u01 of its acceptance draw.  in_prev_row() (is x in t's row?) runs only when it decides.
template <class InPrevRow>
GLT_HD bool node2vec_accept(const Node2VecWeights& w, bool is_prev, float u, InPrevRow in_prev_row) {
  if (is_prev) return u < w.ret;
  if (u < w.lo) return true;
  if (u >= w.hi) return false;
  return in_prev_row() ? u < w.in : u < w.out;
}

}  // namespace glt
