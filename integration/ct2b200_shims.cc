// integration/ct2b200_shims.cc — the reference-side binding of libct2b200.so, COMPILED against the unmodified reference's
// headers (INTEGRATION.md shows the same code as patches to the reference's .cu files).  Each function below is the explicit
// specialisation the reference links today (file:line cited), re-implemented as a call into the C-ABI of include/ct2b200.h.
// Built as its own shared library (oracle/Makefile.shims) and placed in front of the reference's CUDA build, it interposes
// those symbols: the reference's own device-parameterised gtests (tests/ops_test.cc, primitives_test.cc, layers_test.cc) then
// run with the H100 kernels underneath.  Forms the C-ABI does not cover (an axis other than the last, non-transposed rotary
// layouts, ...) are forwarded to the reference's own implementation (dlsym(RTLD_NEXT)), and every call is counted so the
// run reports how many went where.  TEST / INTEGRATION INFRASTRUCTURE: nothing in ctranslate2_b200/ depends on this file.
#include <dlfcn.h>

#include <atomic>
#include <cstdio>
#include <cstdlib>
#include <map>
#include <mutex>
#include <string>

#include <ct2b200.h>

#include "ctranslate2/ops/ops.h"
#include "ctranslate2/primitives.h"
#include "cuda/utils.h"

namespace {

struct Counters {
  std::mutex mu;
  std::map<std::string, std::pair<long, long>> calls;   // name -> {served by ct2b200, forwarded to the reference}
  void hit(const char* name, bool native) {
    std::lock_guard<std::mutex> lock(mu);
    auto& c = calls[name];
    (native ? c.first : c.second)++;
  }
  ~Counters() {
    const char* path = std::getenv("CT2B200_SHIM_REPORT");
    FILE* f = path ? std::fopen(path, "w") : stderr;
    if (!f) f = stderr;
    std::fprintf(f, "ct2b200 shim report (calls served by libct2b200 / forwarded to the reference):\n");
    for (const auto& kv : calls) std::fprintf(f, "  %-44s %8ld %8ld\n", kv.first.c_str(), kv.second.first, kv.second.second);
    if (f != stderr) std::fclose(f);
  }
};
Counters g_counters;

void b200_check(int rc) {
  if (rc == 2) throw std::invalid_argument(ct2b200_last_error());   // shape / argument errors
  if (rc != 0) throw std::runtime_error(ct2b200_last_error());      // CUDA failures (src/cuda/utils.h:51-96)
}

template <typename T> int b200_dtype();
template <> int b200_dtype<float>() { return CT2B200_F32; }
template <> int b200_dtype<ctranslate2::float16_t>() { return CT2B200_F16; }
template <> int b200_dtype<ctranslate2::bfloat16_t>() { return CT2B200_BF16; }

void* stream() { return static_cast<void*>(ctranslate2::cuda::get_cuda_stream()); }

// the reference's own definition of the function that contains `here` (same mangled name, next in the lookup order)
void* next_definition(void* here) {
  Dl_info info;
  if (!dladdr(here, &info) || !info.dli_sname) throw std::runtime_error("ct2b200 shim: cannot name the interposed symbol");
  void* p = dlsym(RTLD_NEXT, info.dli_sname);
  if (!p) throw std::runtime_error(std::string("ct2b200 shim: the reference does not define ") + info.dli_sname);
  return p;
}
#define CT2B200_FORWARD(signature, ...)                                   \
  do {                                                                    \
    __label__ here;                                                       \
  here:                                                                   \
    static void* next = next_definition(&&here);                          \
    using Fn = signature;                                                 \
    return reinterpret_cast<Fn>(next)(__VA_ARGS__);                       \
  } while (0)

}  // namespace

namespace ctranslate2 {

// ---- src/cuda/primitives.cu:571-597 --------------------------------------------------------------------------------
template <>
template <>
void primitives<Device::CUDA>::gemm(bool a_is_packed, bool b_is_packed, bool transpose_a, bool transpose_b, dim_t m, dim_t n,
                                    dim_t k, float alpha, const int8_t* a, dim_t lda, const int8_t* b, dim_t ldb, float beta,
                                    int32_t* c, dim_t ldc, const int32_t* comp) {
  // layers::Dense only ever asks for alpha = 1, beta = 0, trans_b = true and packed leading dimensions
  const bool native = !transpose_a && transpose_b && alpha == 1 && beta == 0 && lda == k && ldb == k && ldc == n && k % 16 == 0;
  g_counters.hit("primitives<CUDA>::gemm<int8,int32>", native);
  if (native) return b200_check(ct2b200_gemm_s8(a, b, m, n, k, c, CT2B200_GEMM_AUTO, stream()));
  CT2B200_FORWARD(void (*)(bool, bool, bool, bool, dim_t, dim_t, dim_t, float, const int8_t*, dim_t, const int8_t*, dim_t, float,
                           int32_t*, dim_t, const int32_t*),
                  a_is_packed, b_is_packed, transpose_a, transpose_b, m, n, k, alpha, a, lda, b, ldb, beta, c, ldc, comp);
}

namespace ops {

// ---- src/ops/quantize_gpu.cu:87-105 ---------------------------------------------------------------------------------
#define SHIM_QUANTIZE(T)                                                                                                  \
  template <>                                                                                                             \
  void Quantize::quantize<Device::CUDA, T, int8_t>(const StorageView& input, StorageView& output, StorageView& scale) const { \
    if (_shift_to_uint8) throw std::invalid_argument("Shift to uin8_t is not defined on CUDA");                          \
    g_counters.hit("Quantize::quantize<CUDA>", true);                                                                    \
    b200_check(ct2b200_quantize_rows(input.data<T>(), b200_dtype<T>(), scale.size(), input.dim(-1), _round_before_cast,   \
                                     output.data<int8_t>(), scale.data<float>(), stream()));                             \
  }
SHIM_QUANTIZE(float)
SHIM_QUANTIZE(float16_t)
SHIM_QUANTIZE(bfloat16_t)

// ---- src/ops/dequantize_gpu.cu:16-27, 96-144 ------------------------------------------------------------------------
#define SHIM_DEQUANTIZE(T)                                                                                                \
  template <>                                                                                                             \
  void Dequantize::dequantize<Device::CUDA, int8_t, T>(const StorageView& input, const StorageView& scale,               \
                                                       StorageView& output) const {                                       \
    g_counters.hit("Dequantize::dequantize<CUDA>", true);                                                                \
    b200_check(ct2b200_dequantize_rows(input.data<int8_t>(), scale.data<float>(), scale.size(), input.dim(-1),           \
                                       output.data<T>(), b200_dtype<T>(), stream()));                                    \
  }                                                                                                                       \
  template <>                                                                                                             \
  void Dequantize::dequantize_gemm_output<Device::CUDA, T>(const StorageView& c, const StorageView& a_scale,             \
                                                           const StorageView& b_scale, const bool transpose_a,           \
                                                           const bool transpose_b, const StorageView* bias,               \
                                                           StorageView& y) const {                                        \
    const bool native = !transpose_a && transpose_b;     /* the only form layers::Dense uses */                          \
    g_counters.hit("Dequantize::dequantize_gemm_output<CUDA>", native);                                                  \
    if (native)                                                                                                           \
      return b200_check(ct2b200_dequantize_gemm_output(c.data<int32_t>(), a_scale.data<float>(), b_scale.data<float>(),   \
                                                       bias ? bias->data<T>() : nullptr,                                  \
                                                       _activation_type ? static_cast<int>(*_activation_type) : -1,      \
                                                       a_scale.size(), c.dim(-1), y.data<T>(), b200_dtype<T>(), stream())); \
    CT2B200_FORWARD(void (*)(const Dequantize*, const StorageView&, const StorageView&, const StorageView&, bool, bool,   \
                             const StorageView*, StorageView&),                                                           \
                    this, c, a_scale, b_scale, transpose_a, transpose_b, bias, y);                                       \
  }
SHIM_DEQUANTIZE(float)
SHIM_DEQUANTIZE(float16_t)
SHIM_DEQUANTIZE(bfloat16_t)

// ---- src/ops/rms_norm_gpu.cu:36-63, layer_norm_gpu.cu:33-66 ---------------------------------------------------------
#define SHIM_NORMS(T)                                                                                                     \
  template <>                                                                                                             \
  void RMSNorm::compute<Device::CUDA, T>(const StorageView& gamma, const StorageView& input, StorageView& output) const { \
    const dim_t depth = input.dim(-1);                                                                                    \
    g_counters.hit("RMSNorm::compute<CUDA>", true);                                                                      \
    b200_check(ct2b200_rms_norm(gamma.data<T>(), input.data<T>(), input.size() / depth, depth, _epsilon, _use_residual,   \
                                output.data<T>(), b200_dtype<T>(), stream()));                                           \
  }                                                                                                                       \
  template <>                                                                                                             \
  void LayerNorm::compute<Device::CUDA, T>(const StorageView* beta, const StorageView* gamma, const StorageView& input,   \
                                           const dim_t axis, const dim_t outer_size, const dim_t axis_size,               \
                                           const dim_t inner_size, StorageView& output) const {                           \
    const bool native = axis == input.rank() - 1;                                                                        \
    g_counters.hit("LayerNorm::compute<CUDA>", native);                                                                  \
    if (native)                                                                                                           \
      return b200_check(ct2b200_layer_norm(input.data<T>(), gamma ? gamma->data<T>() : nullptr,                           \
                                           beta ? beta->data<T>() : nullptr, outer_size, axis_size, _epsilon,             \
                                           output.data<T>(), nullptr, nullptr, 1, b200_dtype<T>(), stream()));           \
    CT2B200_FORWARD(void (*)(const LayerNorm*, const StorageView*, const StorageView*, const StorageView&, dim_t, dim_t, dim_t, \
                             dim_t, StorageView&),                                                                        \
                    this, beta, gamma, input, axis, outer_size, axis_size, inner_size, output);                          \
  }
SHIM_NORMS(float)
SHIM_NORMS(float16_t)
SHIM_NORMS(bfloat16_t)

// ---- src/ops/rotary_gpu.cu:57-85, softmax_gpu.cu:17-31, topk_gpu.cu:27-55, gather_gpu.cu:52-91 ---------------------------
#define SHIM_ROW_OPS(T)                                                                                                   \
  template <>                                                                                                             \
  void Rotary::compute<Device::CUDA, T>(const StorageView& input, const StorageView& sin, const StorageView& cos,         \
                                        StorageView& output, bool is_transposed) const {                                  \
    g_counters.hit("Rotary::compute<CUDA>", is_transposed);                                                              \
    if (is_transposed) {  /* [batch, heads, time, depth]: rows = batch * heads sequences of `time` positions */          \
      const dim_t depth = input.dim(-1), time = input.dim(-2);                                                            \
      return b200_check(ct2b200_rotary(input.data<T>(), sin.data<T>(), cos.data<T>(), input.size() / (time * depth), time, \
                                       depth, _ndims == 0 ? depth : _ndims, _interleave, output.data<T>(), b200_dtype<T>(), \
                                       stream()));                                                                        \
    }                                                                                                                     \
    CT2B200_FORWARD(void (*)(const Rotary*, const StorageView&, const StorageView&, const StorageView&, StorageView&, bool), \
                    this, input, sin, cos, output, is_transposed);                                                       \
  }                                                                                                                       \
  template <>                                                                                                             \
  void SoftMax::compute<Device::CUDA, T>(const StorageView& input, const StorageView* lengths, StorageView& output) const { \
    const dim_t depth = input.dim(-1);                                                                                    \
    g_counters.hit("SoftMax::compute<CUDA>", true);                                                                      \
    b200_check(ct2b200_softmax(input.data<T>(), lengths ? lengths->data<int32_t>() : nullptr, input.size() / depth, depth, \
                               _log, output.data<T>(), b200_dtype<T>(), stream()));                                      \
  }                                                                                                                       \
  template <>                                                                                                             \
  void TopK::compute<Device::CUDA, T, int32_t>(const StorageView& x, StorageView& values, StorageView& indices) const {   \
    const dim_t depth = x.dim(-1);                                                                                        \
    const bool native = _k <= 64;                                                                                         \
    g_counters.hit("TopK::compute<CUDA>", native);                                                                       \
    if (native)                                                                                                           \
      return b200_check(ct2b200_topk(x.data<T>(), x.size() / depth, depth, static_cast<int>(_k), values.data<T>(),        \
                                     indices.data<int32_t>(), b200_dtype<T>(), stream()));                               \
    CT2B200_FORWARD(void (*)(const TopK*, const StorageView&, StorageView&, StorageView&), this, x, values, indices);      \
  }                                                                                                                       \
  template <>                                                                                                             \
  void Gather::compute<Device::CUDA, T>(const StorageView& data, const StorageView& input, const dim_t axis,              \
                                        const dim_t batch_dims, StorageView& output) const {                              \
    const bool native = axis == 0 && batch_dims == 0;                                                                     \
    g_counters.hit("Gather::compute<CUDA>", native);                                                                     \
    if (native)                                                                                                           \
      return b200_check(ct2b200_gather_rows(data.data<T>(), input.data<int32_t>(), input.size(),                          \
                                            data.stride(0) * static_cast<dim_t>(sizeof(T)), output.data<T>(), stream())); \
    CT2B200_FORWARD(void (*)(const Gather*, const StorageView&, const StorageView&, dim_t, dim_t, StorageView&), this, data, \
                    input, axis, batch_dims, output);                                                                     \
  }
SHIM_ROW_OPS(float)
SHIM_ROW_OPS(float16_t)
SHIM_ROW_OPS(bfloat16_t)

}  // namespace ops
}  // namespace ctranslate2
