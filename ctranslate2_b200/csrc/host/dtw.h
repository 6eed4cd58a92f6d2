// dtw.h — negative_dtw + backtrace of the reference (src/dtw.cc), host only: the alignment path through a [n, m] matrix that
// maximises the summed values.  Ties follow the reference exactly: diagonal only if strictly below both, up only if strictly
// below both, otherwise left (which is also where NaN comparisons fall).  Shared by Translator::whisper_align and the C-ABI
// ct2b200_negative_dtw_host.
#pragma once

#include <algorithm>
#include <cstdint>
#include <limits>
#include <stdexcept>
#include <utility>
#include <vector>

namespace ct2b200 {

// x [n, m] row-major; returns the (row, column) pairs from the start, (-1) entries included where the reference yields them
inline std::vector<std::pair<int64_t, int64_t>> negative_dtw(const float* x, int64_t n, int64_t m) {
  const float inf = std::numeric_limits<float>::infinity();
  std::vector<float> cost((n + 1) * (m + 1), inf);
  std::vector<int8_t> trace((n + 1) * (m + 1), -1);
  auto C = [&](int64_t i, int64_t j) -> float& { return cost[i * (m + 1) + j]; };
  auto Tr = [&](int64_t i, int64_t j) -> int8_t& { return trace[i * (m + 1) + j]; };
  C(0, 0) = 0.f;
  for (int64_t j = 1; j < m + 1; ++j)
    for (int64_t i = 1; i < n + 1; ++i) {
      const float c0 = C(i - 1, j - 1), c1 = C(i - 1, j), c2 = C(i, j - 1);
      float c;
      int8_t t;
      if (c0 < c1 && c0 < c2) {
        c = c0;
        t = 0;
      } else if (c1 < c0 && c1 < c2) {
        c = c1;
        t = 1;
      } else {
        c = c2;
        t = 2;
      }
      C(i, j) = -x[(i - 1) * m + (j - 1)] + c;
      Tr(i, j) = t;
    }
  // backtrace (dtw.cc:8-38)
  int64_t i = n, j = m;
  for (int64_t k = 0; k <= j; ++k) Tr(0, k) = 2;
  for (int64_t k = 0; k <= i; ++k) Tr(k, 0) = 1;
  std::vector<std::pair<int64_t, int64_t>> path;
  while (i > 0 || j > 0) {
    path.emplace_back(i - 1, j - 1);
    const int t = Tr(i, j);
    if (t == 0) {
      --i;
      --j;
    } else if (t == 1) {
      --i;
    } else if (t == 2) {
      --j;
    } else {
      throw std::runtime_error("Unexpected trace[i, j]");
    }
  }
  std::reverse(path.begin(), path.end());
  return path;
}

}  // namespace ct2b200
