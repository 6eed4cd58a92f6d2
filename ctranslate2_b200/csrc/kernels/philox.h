// philox.h — Philox4x32-10 (Salmon, Moraes, Dror, Shaw, "Parallel random numbers: as easy as 1, 2, 3", SC 2011), written from
// the published algorithm as plain code shared by the sampling kernels (seq2seq.cu, sample_row.cuh) and a host entry point
// (ct2b200_philox4x32_host) that lets the CPU test suite check it against known-answer vectors.
//
// The uniform of one draw: u = (word 0 of Philox4x32-10(counter, key) >> 8) * 2^-24, in [0, 1) with 24 bits, where
//   counter = {step, row, call, 0}, key = {seed, 0}
// for (process seed, sampling call index, decoder row, absolute decoding step).  Distinct (call, row, step) never share a block.
#pragma once

#include <cstdint>

#ifndef CT2B200_HD
#if defined(__CUDACC__)
#define CT2B200_HD __host__ __device__
#else
#define CT2B200_HD
#endif
#endif

namespace ct2b200 {

struct Philox4 {
  uint32_t v[4];
};

CT2B200_HD inline void philox_mulhilo(uint32_t a, uint32_t b, uint32_t& hi, uint32_t& lo) {
  const uint64_t p = static_cast<uint64_t>(a) * b;
  hi = static_cast<uint32_t>(p >> 32);
  lo = static_cast<uint32_t>(p);
}

CT2B200_HD inline Philox4 philox4x32_10(Philox4 c, uint32_t k0, uint32_t k1) {
  for (int r = 0; r < 10; ++r) {
    if (r > 0) {
      k0 += 0x9E3779B9u;
      k1 += 0xBB67AE85u;
    }
    uint32_t hi0, lo0, hi1, lo1;
    philox_mulhilo(0xD2511F53u, c.v[0], hi0, lo0);
    philox_mulhilo(0xCD9E8D57u, c.v[2], hi1, lo1);
    c = Philox4{{hi1 ^ c.v[1] ^ k0, lo1, hi0 ^ c.v[3] ^ k1, lo0}};
  }
  return c;
}

CT2B200_HD inline float philox_uniform(uint32_t seed, uint32_t call, uint32_t row, uint32_t step) {
  const Philox4 r = philox4x32_10(Philox4{{step, row, call, 0u}}, seed, 0u);
  return static_cast<float>(r.v[0] >> 8) * (1.f / 16777216.f);
}

}  // namespace ct2b200
