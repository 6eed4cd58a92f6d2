// engine.cc — host side: model.bin loader, Llama-class decoder driver, greedy search, Generator.
// See engine.h.  Reference counterparts: src/models/model.cc, src/layers/{transformer,attention,common}.cc,
// src/decoding.cc, src/models/language_model.cc, src/generator.cc.
#include "engine.h"

#include "beam.h"


#include <cuda_profiler_api.h>
#include <fcntl.h>
#include <sys/mman.h>
#include <sys/stat.h>
#include <unistd.h>

#include <algorithm>
#include <cmath>
#include <cstdlib>
#include <cstring>
#include <tuple>
#include <fstream>
#include <sstream>

namespace ct2b200 {

// =============================================================================================
// ModelFile
// =============================================================================================
namespace {
struct Cursor {
  const uint8_t* p;
  const uint8_t* end;
  template <typename U> U read() {
    if (p + sizeof(U) > end) throw std::runtime_error("model.bin: unexpected end of file");
    U v;
    std::memcpy(&v, p, sizeof(U));
    p += sizeof(U);
    return v;
  }
  std::string read_string() {
    const uint16_t n = read<uint16_t>();
    if (p + n > end) throw std::runtime_error("model.bin: unexpected end of file");
    std::string s(reinterpret_cast<const char*>(p), n ? n - 1 : 0);
    p += n;
    return s;
  }
};
size_t type_size(int type_id) {
  switch (type_id) {
    case 0: return 4;   // float32
    case 1: return 1;   // int8
    case 2: return 2;   // int16
    case 3: return 4;   // int32
    case 4: return 2;   // float16
    case 5: return 2;   // bfloat16
    default: throw std::runtime_error("model.bin: unknown data type id " + std::to_string(type_id));
  }
}
float half_bits_to_float(uint16_t h) {
  const uint32_t sign = (h >> 15) & 1, exp = (h >> 10) & 0x1F, man = h & 0x3FF;
  float v;
  if (exp == 0) v = std::ldexp(static_cast<float>(man), -24);
  else if (exp == 31) v = man ? NAN : INFINITY;
  else v = std::ldexp(static_cast<float>(man | 0x400), static_cast<int>(exp) - 25);
  return sign ? -v : v;
}
float bf16_bits_to_float(uint16_t b) {
  uint32_t u = static_cast<uint32_t>(b) << 16;
  float f;
  std::memcpy(&f, &u, 4);
  return f;
}
}  // namespace

double HostVariable::scalar() const {
  switch (type_id) {
    case 0: { float v; std::memcpy(&v, data, 4); return v; }
    case 1: return *reinterpret_cast<const int8_t*>(data);
    case 2: { int16_t v; std::memcpy(&v, data, 2); return v; }
    case 3: { int32_t v; std::memcpy(&v, data, 4); return v; }
    case 4: { uint16_t v; std::memcpy(&v, data, 2); return half_bits_to_float(v); }
    default: { uint16_t v; std::memcpy(&v, data, 2); return bf16_bits_to_float(v); }
  }
}

ModelFile::ModelFile(const std::string& model_dir) {
  const std::string path = model_dir + "/model.bin";
  const int fd = ::open(path.c_str(), O_RDONLY);
  if (fd < 0) throw std::runtime_error("Unable to open file 'model.bin' in model '" + model_dir + "'");
  struct stat st;
  ::fstat(fd, &st);
  map_size_ = static_cast<size_t>(st.st_size);
  map_ = ::mmap(nullptr, map_size_, PROT_READ, MAP_PRIVATE, fd, 0);
  ::close(fd);
  if (map_ == MAP_FAILED) throw std::runtime_error("mmap failed for " + path);
  Cursor c{static_cast<const uint8_t*>(map_), static_cast<const uint8_t*>(map_) + map_size_};
  binary_version = c.read<uint32_t>();
  if (binary_version < 2 || binary_version > 6)
    throw std::runtime_error("Unsupported model binary version " + std::to_string(binary_version) +
                             " (this engine reads versions 2 to 6)");
  spec_name = c.read_string();
  revision = c.read<uint32_t>();
  const uint32_t nvars = c.read<uint32_t>();
  for (uint32_t i = 0; i < nvars; ++i) {
    const std::string name = c.read_string();
    HostVariable v;
    const uint8_t rank = c.read<uint8_t>();
    for (int r = 0; r < rank; ++r) v.shape.push_back(c.read<uint32_t>());
    if (binary_version >= 4) {
      v.type_id = c.read<uint8_t>();
      v.nbytes = c.read<uint32_t>();
    } else {
      // versions 2-3 store the item size and the item count (model.cc:653-657, get_dtype_from_item_size)
      const uint8_t item_size = c.read<uint8_t>();
      v.type_id = item_size == 4 ? 0 : item_size == 2 ? 2 : item_size == 1 ? 1 : -1;
      if (v.type_id < 0) throw std::runtime_error("model.bin: unknown item size " + std::to_string(item_size));
      v.nbytes = static_cast<size_t>(c.read<uint32_t>()) * item_size;
    }
    if (static_cast<size_t>(v.size()) * type_size(v.type_id) != v.nbytes)
      throw std::runtime_error("model.bin: variable " + name + " has inconsistent size");
    if (c.p + v.nbytes > c.end) throw std::runtime_error("model.bin: unexpected end of file");
    v.data = c.p;
    c.p += v.nbytes;
    vars_.emplace(name, v);
  }
  const uint32_t naliases = binary_version >= 3 ? c.read<uint32_t>() : 0;
  for (uint32_t i = 0; i < naliases; ++i) {
    const std::string alias = c.read_string();
    const std::string target = c.read_string();
    auto it = vars_.find(target);
    if (it == vars_.end()) throw std::runtime_error("model.bin: alias target not found: " + target);
    vars_.emplace(alias, it->second);
    // the quantization scale / zero of the target follows its alias (model.cc:772-774)
    for (const char* suffix : {"_scale", "_zero"}) {
      auto sit = vars_.find(target + suffix);
      if (sit != vars_.end()) vars_.emplace(alias + suffix, sit->second);
    }
  }
  std::ifstream cf(model_dir + "/config.json");
  if (cf) {
    std::stringstream ss;
    ss << cf.rdbuf();
    config_json_ = ss.str();
  }
}

ModelFile::~ModelFile() {
  if (map_ && map_ != MAP_FAILED) ::munmap(map_, map_size_);
}

const HostVariable* ModelFile::find(const std::string& name) const {
  auto it = vars_.find(name);
  return it == vars_.end() ? nullptr : &it->second;
}
const HostVariable& ModelFile::get(const std::string& name) const {
  const HostVariable* v = find(name);
  if (!v) throw std::out_of_range("variable " + name + " not found");   // models/model.cc get_variable
  return *v;
}
double ModelFile::attribute(const std::string& name, double fallback) const {
  const HostVariable* v = find(name);
  return v ? v->scalar() : fallback;
}
double ModelFile::config_number(const std::string& key, double fallback) const {
  const std::string needle = "\"" + key + "\"";
  size_t pos = config_json_.find(needle);
  if (pos == std::string::npos) return fallback;
  pos = config_json_.find(':', pos);
  if (pos == std::string::npos) return fallback;
  const char* s = config_json_.c_str() + pos + 1;
  char* e = nullptr;
  const double v = std::strtod(s, &e);
  return e == s ? fallback : v;   // null / non-number -> fallback
}

// =============================================================================================
// device buffers
// =============================================================================================
void DeviceBuffer::alloc(size_t n) {
  release();
  if (n == 0) return;
  CT2_CUDA_CHECK(cudaMalloc(&ptr, n));
  bytes = n;
}
void DeviceBuffer::release() {
  if (ptr) cudaFree(ptr);
  ptr = nullptr;
  bytes = 0;
}

void StepGraph::reset() {
  if (exec) cudaGraphExecDestroy(exec);
  exec = nullptr;
  nodes = 0;
  key.clear();
}

void StepGraph::capture(cudaStream_t st, const std::vector<int64_t>& k, const std::function<void()>& step) {
  if (exec && key == k) return;
  reset();
  cudaGraph_t g = nullptr;
  const int64_t before = g_kernel_launches.load();
  CT2_CUDA_CHECK(cudaStreamBeginCapture(st, cudaStreamCaptureModeThreadLocal));
  try {
    step();
  } catch (...) {
    cudaStreamEndCapture(st, &g);
    if (g) cudaGraphDestroy(g);
    throw;
  }
  CT2_CUDA_CHECK(cudaStreamEndCapture(st, &g));
  g_kernel_launches.store(before);     // captured launches are counted when the graph is replayed
  size_t n = 0;
  cudaGraphGetNodes(g, nullptr, &n);
  nodes = static_cast<int64_t>(n);
  CT2_CUDA_CHECK(cudaGraphInstantiate(&exec, g, 0));
  cudaGraphDestroy(g);
  key = k;
}

void StepGraph::launch(cudaStream_t st) {
  CT2_CUDA_CHECK(cudaGraphLaunch(exec, st));
  count_launch(static_cast<int>(nodes));
}

int64_t eos_poll_interval() {
  const char* env = std::getenv("CT2B200_EOS_POLL");
  return std::max<int64_t>(1, env ? std::atoll(env) : 4);
}

// host-side conversion of a float-ish variable to the compute dtype
std::vector<uint8_t> convert_to_dtype(const HostVariable& v, int dtype) {
  const int64_t n = v.size();
  std::vector<float> f(n);
  for (int64_t i = 0; i < n; ++i) {
    switch (v.type_id) {
      case 0: std::memcpy(&f[i], v.data + 4 * i, 4); break;
      case 4: { uint16_t h; std::memcpy(&h, v.data + 2 * i, 2); f[i] = half_bits_to_float(h); break; }
      case 5: { uint16_t h; std::memcpy(&h, v.data + 2 * i, 2); f[i] = bf16_bits_to_float(h); break; }
      default: throw std::runtime_error("expected a floating point variable");
    }
  }
  std::vector<uint8_t> out(n * dtype_size(dtype));
  if (dtype == CT2B200_F32) {
    std::memcpy(out.data(), f.data(), n * 4);
  } else if (dtype == CT2B200_F16) {
    for (int64_t i = 0; i < n; ++i) {
      const __half h = __float2half_rn(f[i]);
      std::memcpy(out.data() + 2 * i, &h, 2);
    }
  } else {
    for (int64_t i = 0; i < n; ++i) {
      const __nv_bfloat16 h = __float2bfloat16_rn(f[i]);
      std::memcpy(out.data() + 2 * i, &h, 2);
    }
  }
  return out;
}

// Host (pageable: the model file) -> device.  cudaMemcpy may return once the data sits in the driver's staging buffer, BEFORE the
// DMA into `dst` has finished; the kernels and device-to-device copies that follow run on the engine's own non-blocking stream,
// which does not wait for the legacy stream.  Without the synchronisation the tensor-parallel shard cut right after the upload
// can read a partly written matrix (tests/tp_worker.py).
void upload(DeviceBuffer& dst, const void* src, size_t n) {
  dst.alloc(n);
  if (n) {
    CT2_CUDA_CHECK(cudaMemcpy(dst.ptr, src, n, cudaMemcpyHostToDevice));
    CT2_CUDA_CHECK(cudaDeviceSynchronize());
  }
}

namespace {

int env_gemm_impl() {
  const char* e = std::getenv("CT2B200_GEMM_IMPL");
  if (!e) return CT2B200_GEMM_AUTO;
  if (std::strcmp(e, "mma") == 0) return CT2B200_GEMM_MMA_SYNC;
  if (std::strcmp(e, "tc") == 0 || std::strcmp(e, "tcgen05") == 0) return CT2B200_GEMM_TCGEN05;
  return CT2B200_GEMM_AUTO;
}

}  // namespace

// ct2b200_gemm_impl dispatch.  AUTO = wgmma (the sm_90a path); mma.sync only on request.
void gemm_s8(const int8_t* A, const int8_t* B, int64_t M, int64_t N, int64_t K, const DenseEpilogue& epi,
             int dtype, int impl, cudaStream_t st) {
  if (impl == CT2B200_GEMM_AUTO) impl = env_gemm_impl();
  if (impl == CT2B200_GEMM_MMA_SYNC) gemm_s8_mma(A, B, M, N, K, epi, dtype, st);
  else gemm_s8_tc(A, B, M, N, K, epi, dtype, st);
}
// float Dense (ops::Gemm float arms, primitives.cu:485-569): f16 / bf16 on wgmma kind::f16, f32 as true fp32 FMAs
void gemm_float(const void* A, const void* B, const void* bias, const void* residual, int act, int64_t M, int64_t N,
                int64_t K, void* C, int dtype, cudaStream_t st) {
  if (dtype == CT2B200_F32)
    gemm_f32(static_cast<const float*>(A), static_cast<const float*>(B), static_cast<const float*>(bias),
             static_cast<const float*>(residual), act, M, N, K, static_cast<float*>(C), st);
  else
    gemm_f16_tc(A, B, bias, residual, act, M, N, K, C, dtype, st);
}
void gemm_s8_glu(const int8_t* A, const int8_t* Bgate, const int8_t* Bup, int64_t M, int64_t N, int64_t K,
                 const GluEpilogue& glu, int dtype, int impl, cudaStream_t st) {
  if (impl == CT2B200_GEMM_AUTO) impl = env_gemm_impl();
  if (impl == CT2B200_GEMM_MMA_SYNC) gemm_s8_glu_mma(A, Bgate, Bup, M, N, K, glu, dtype, st);
  else gemm_s8_glu_tc(A, Bgate, Bup, M, N, K, glu, dtype, st);
}

size_t upload_as(DeviceBuffer& dst, const HostVariable& v, int dtype) {
  const auto bytes = convert_to_dtype(v, dtype);
  upload(dst, bytes.data(), bytes.size());
  return bytes.size();
}

EngineDevice::EngineDevice(int dev) : device(dev) {
  CT2_CUDA_CHECK(cudaSetDevice(device));
  int major = 0;
  CT2_CUDA_CHECK(cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, device));
  if (major != 9)
    throw std::runtime_error("ct2b200 is built for sm_90a (H100); found compute capability major " + std::to_string(major));
  CT2_CUDA_CHECK(cudaDeviceGetAttribute(&sm_count, cudaDevAttrMultiProcessorCount, device));
  CT2_CUDA_CHECK(cudaStreamCreateWithFlags(&stream, cudaStreamNonBlocking));
  SplitKWorkspace::get(stream);
}

EngineDevice::~EngineDevice() {
  cudaSetDevice(device);   // the workspace is registered per (device, stream)
  cudaStreamSynchronize(stream);
  SplitKWorkspace::release(stream);
  cudaStreamDestroy(stream);
}

// =============================================================================================
// Dense layers: loading, tensor-parallel cut, dispatch
// =============================================================================================
namespace {
// rows [b, e) of a dimension split evenly over the tensor-parallel ranks
std::pair<int64_t, int64_t> shard_range(int64_t total, int rank, int world) {
  CT2_REQUIRE(total % world == 0, "tensor parallel: dimension is not divisible by the number of ranks");
  const int64_t per = total / world;
  return {rank * per, (rank + 1) * per};
}
}  // namespace

int64_t ShardPlan::n() const {
  int64_t n = 0;
  for (const auto& r : rows) n += r.second - r.first;
  return n;
}

ShardPlan shard_plan(Shard shard, int64_t n, int64_t k, int heads, int heads_kv, int head_dim, int rank, int world,
                     int64_t group) {
  ShardPlan p;
  p.rows = {{0, n}};
  p.k1 = k;
  if (world == 1 || shard == Shard::REPLICATED) return p;
  if (shard == Shard::ROWS) {
    p.rows = {shard_range(n, rank, world)};
  } else if (shard == Shard::QKV_ROWS) {
    const int64_t D = head_dim, hq = static_cast<int64_t>(heads) * D, hk = static_cast<int64_t>(heads_kv) * D;
    CT2_REQUIRE(n == hq + 2 * hk, "fused QKV weight has an unexpected number of rows");
    const auto q = shard_range(heads, rank, world), kv = shard_range(heads_kv, rank, world);
    p.rows = {{q.first * D, q.second * D}, {hq + kv.first * D, hq + kv.second * D},
              {hq + hk + kv.first * D, hq + hk + kv.second * D}};
  } else {
    std::tie(p.k0, p.k1) = shard_range(k, rank, world);
    CT2_REQUIRE(group == 0 || (p.k0 % group == 0 && p.k1 % group == 0),
                "tensor parallel: the AWQ group size must divide the K slice");
  }
  return p;
}

namespace {
// One channel-major buffer of a Dense layer: `bytes` per `per_k` input columns of an output row, or per output row when
// per_k == 0 (a value per output channel, not split along K).
struct ShardCut {
  DeviceBuffer* buf;
  int64_t bytes, per_k;
};

// Replaces every non-empty buffer by its rows and K range of `plan` (k = the unsharded K), device to device.  The values are
// those of the unsharded layer (int8 values and their per-channel scales included), so the shards reproduce the single-GPU
// arithmetic.
void cut_shard(const ShardPlan& plan, int64_t k, cudaStream_t st, std::initializer_list<ShardCut> parts) {
  std::vector<DeviceBuffer> cut;
  cut.reserve(parts.size());
  for (const ShardCut& c : parts) {
    if (!c.buf->ptr) {
      cut.emplace_back();
      continue;
    }
    const int64_t pitch = c.per_k ? k / c.per_k * c.bytes : c.bytes;
    const int64_t width = c.per_k ? plan.k() / c.per_k * c.bytes : c.bytes;
    const int64_t skip = c.per_k ? plan.k0 / c.per_k * c.bytes : 0;
    cut.emplace_back(static_cast<size_t>(plan.n()) * width);
    int64_t o = 0;
    for (const auto& r : plan.rows) {
      CT2_CUDA_CHECK(cudaMemcpy2DAsync(cut.back().as<uint8_t>() + o * width, width, c.buf->as<uint8_t>() + r.first * pitch + skip,
                                       pitch, width, r.second - r.first, cudaMemcpyDeviceToDevice, st));
      o += r.second - r.first;
    }
  }
  CT2_CUDA_CHECK(cudaStreamSynchronize(st));
  auto it = cut.begin();
  for (const ShardCut& c : parts) {
    if (c.buf->ptr) *c.buf = std::move(*it);
    ++it;
  }
}

// The matrix of a Dense layer as the requested arithmetic wants it: Model::set_compute_type + ensure_dtype
// (src/models/model.cc:178-234, 304-369) on the GPU.  The stored matrix goes to the device as it is; when the compute type
// asks for another weight type it is converted there with the converter's own arithmetic (model_spec.py:222-243 =
// ops::Quantize on fp32: scale = 127 / amax per row, q = rint(w * scale); back: w = T(float(q) * (1 / scale)),
// dequantize_cpu.cc:12-21).  The result is int8 + fp32 row scales (INT8) or T [N, K] (FLOAT16).
void load_matrix(const ModelFile& f, const std::string& prefix, const DenseLoad& o, DenseWeights& w) {
  const HostVariable& wt = f.get(prefix + "/weight");
  CT2_REQUIRE(wt.type_id == 1 || wt.type_id == 0 || wt.type_id == 4 || wt.type_id == 5, "unsupported weight type for " + prefix);
  CT2_REQUIRE(wt.shape.size() == 2, "weight must be a matrix");
  const int64_t N = wt.shape[0], K = wt.shape[1];
  const bool stored_int8 = wt.type_id == 1;
  const bool want_int8 = o.weight_type == CT2B200_WEIGHTS_INT8 || (o.weight_type == CT2B200_WEIGHTS_STORED && stored_int8);
  w.kind = want_int8 ? DenseWeights::INT8 : DenseWeights::FLOAT16;
  w.n = N;
  w.k = K;
  if (stored_int8) {
    const HostVariable& sc = f.get(prefix + "/weight_scale");
    CT2_REQUIRE(sc.type_id == 0 && sc.size() == N, "weight_scale must be float32 [n]");
    upload(w.weight, wt.data, wt.nbytes);
    upload(w.scale, sc.data, sc.nbytes);
    if (!want_int8) {                            // int8 -> float (compute types float16 / bfloat16 on an int8 model)
      DeviceBuffer deq(static_cast<size_t>(N) * K * dtype_size(o.dtype));
      launch_dequantize_rows(w.weight.as<int8_t>(), w.scale.as<float>(), N, K, deq.ptr, o.dtype, o.stream, /*reciprocal=*/true);
      CT2_CUDA_CHECK(cudaStreamSynchronize(o.stream));
      w.weight = std::move(deq);
      w.scale.release();
    }
  } else {
    const int stored = wt.type_id == 0 ? CT2B200_F32 : wt.type_id == 4 ? CT2B200_F16 : CT2B200_BF16;
    upload(w.weight, wt.data, wt.nbytes);
    if (want_int8 || stored != o.dtype) {
      DeviceBuffer f32;
      const float* src32 = w.weight.as<float>();
      if (stored != CT2B200_F32) {
        f32.alloc(static_cast<size_t>(N) * K * 4);
        launch_convert_to_f32(w.weight.ptr, N * K, f32.as<float>(), stored, o.stream);
        src32 = f32.as<float>();
      }
      if (want_int8) {                           // float -> int8 (e.g. a float16 model served as int8_float16)
        DeviceBuffer q(static_cast<size_t>(N) * K);
        w.scale.alloc(static_cast<size_t>(N) * 4);
        launch_quantize_rows(src32, CT2B200_F32, N, K, true, q.as<int8_t>(), w.scale.as<float>(), o.stream);
        CT2_CUDA_CHECK(cudaStreamSynchronize(o.stream));
        w.weight = std::move(q);
      } else {                                   // float -> the compute float type
        DeviceBuffer t(static_cast<size_t>(N) * K * dtype_size(o.dtype));
        launch_convert_from_f32(src32, N * K, t.ptr, o.dtype, o.stream);
        CT2_CUDA_CHECK(cudaStreamSynchronize(o.stream));
        w.weight = std::move(t);
      }
    }
  }
}

// AWQ-INT4 (model.cc:750-757 pins FLOAT16): repacked once into the native channel-major layout (kernels/awq.cu)
void load_awq(const ModelFile& f, const std::string& prefix, const DenseLoad& o, DenseWeights& w) {
  CT2_REQUIRE(o.dtype == CT2B200_F16, "AWQ models run with float16 activations (the reference forces ComputeType::FLOAT16)");
  const int layout = static_cast<int>(f.config_number("quantization_type", 0));
  CT2_REQUIRE(layout == 1 || layout == 2, "config.json quantization_type must be 1 (AWQ_GEMM) or 2 (AWQ_GEMV)");
  const HostVariable& wt = f.get(prefix + "/weight");
  const HostVariable& sc = f.get(prefix + "/weight_scale");
  const HostVariable& zr = f.get(prefix + "/weight_zero");
  CT2_REQUIRE(sc.type_id == 4, "AWQ scales must be float16");
  w.kind = layout == 1 ? DenseWeights::AWQ_GEMM : DenseWeights::AWQ_GEMV;
  if (layout == 1) {            // qweight [K, N/8], scales [K/G, N]
    w.k = wt.shape[0];
    w.n = wt.shape[1] * 8;
    w.group_size = static_cast<int>(w.k / sc.shape[0]);
  } else {                      // qweight [N, K/8], scales [N, K/G (padded)]
    w.n = wt.shape[0];
    w.k = wt.shape[1] * 8;
    const int g = static_cast<int>(f.config_number("quantization_group_size", 128));
    w.group_size = g > 0 ? g : 128;
  }
  DeviceBuffer qw, qs, qz;
  upload(qw, wt.data, wt.nbytes);
  upload(qs, sc.data, sc.nbytes);
  upload(qz, zr.data, zr.nbytes);
  const int64_t ng = w.k / w.group_size;
  w.weight.alloc(static_cast<size_t>(w.n) * (w.k / 8) * 4);
  w.scale.alloc(static_cast<size_t>(w.n) * ng * 2);
  w.zeros.alloc(static_cast<size_t>(w.n) * ng * 2);
  awq_repack(qw.as<int32_t>(), qs.ptr, qz.as<int32_t>(), layout, w.group_size, w.n, w.k, w.weight.as<int32_t>(),
             w.scale.ptr, w.zeros.ptr, o.stream);
  CT2_CUDA_CHECK(cudaStreamSynchronize(o.stream));
}
}  // namespace

int64_t load_dense(const ModelFile& f, const std::string& prefix, const DenseLoad& o, DenseWeights& w) {
  const HostVariable& wt = f.get(prefix + "/weight");
  const bool awq = o.awq && wt.type_id == 3 && f.find(prefix + "/weight_zero") != nullptr;
  if (awq) load_awq(f, prefix, o, w);
  else load_matrix(f, prefix, o, w);
  const bool sharded = o.world > 1 && o.shard != Shard::REPLICATED;
  if (const HostVariable* b = f.find(prefix + "/bias")) {
    // row-parallel: the whole bias on rank 0 only (common.cc:348-352); column-parallel: its rows are cut with the weight
    CT2_REQUIRE(!(awq && sharded), "tensor parallel: biased AWQ layers are not sharded");
    if (!sharded || o.shard != Shard::COLS || o.rank == 0) upload_as(w.bias, *b, o.dtype);
  }
  // Tensor-parallel shards (model.cc:662-743) are cut from the converted (channel-major) tensors
  const ShardPlan plan = shard_plan(o.shard, w.n, w.k, o.heads, o.heads_kv, o.head_dim, o.rank, o.world, awq ? w.group_size : 0);
  if (sharded) {
    const int64_t G = w.group_size, es = static_cast<int64_t>(dtype_size(o.dtype));
    if (awq)                                     // 8 K per packed int32 word, one f16 scale / zero per group
      cut_shard(plan, w.k, o.stream, {{&w.weight, 4, 8}, {&w.scale, 2, G}, {&w.zeros, 2, G}});
    else if (w.kind == DenseWeights::INT8)
      cut_shard(plan, w.k, o.stream, {{&w.weight, 1, 1}, {&w.scale, 4, 0}, {&w.bias, es, 0}});
    else
      cut_shard(plan, w.k, o.stream, {{&w.weight, es, 1}, {&w.bias, es, 0}});
    w.n = plan.n();
    w.k = plan.k();
  }
  if (awq) {
    // group-major {scale, zero} pairs for the decode kernel (coalesced fetches); the channel-major arrays stay for the
    // general kernel, the prompt-pass dequantisation and the op-level API
    const AwqNative a = awq_view(w);
    w.scale_zero.alloc(static_cast<size_t>(w.n) * (w.k / w.group_size) * 4);
    awq_build_group_major(a, w.scale_zero.ptr, o.stream);
    CT2_CUDA_CHECK(cudaStreamSynchronize(o.stream));
  }
  return static_cast<int64_t>(w.weight.bytes + w.scale.bytes + w.zeros.bytes);
}

AwqNative awq_view(const DenseWeights& w) {
  return {w.weight.ptr, w.scale.ptr, w.zeros.ptr, w.n, w.k, w.group_size, w.scale_zero.ptr};
}

void rows_to_int8(const void* x, const void* gamma, float eps, int64_t m, int64_t k, int dtype, int8_t* xq, float* xs,
                  cudaStream_t st) {
  if (gamma) launch_rms_norm(gamma, x, m, k, eps, false, nullptr, xq, xs, dtype, st);
  else launch_quantize_rows(x, dtype, m, k, true, xq, xs, st);
}

void dense_forward(const DenseWeights& w, const int8_t* xq, const float* xs, const void* x, int64_t m, const void* residual,
                   int act, void* y, int64_t ldy, int dtype, int gemm_impl, void* awq_scratch, cudaStream_t st) {
  if (ldy == 0) ldy = w.n;
  if (w.kind == DenseWeights::INT8) {
    DenseEpilogue e{xs, w.scale.as<float>(), w.bias.ptr, residual, y, nullptr, act, ldy};
    gemm_s8(xq, w.weight.as<int8_t>(), m, w.n, w.k, e, dtype, gemm_impl, st);
    return;
  }
  CT2_REQUIRE(ldy == w.n, "float Dense writes contiguous rows");
  if (w.kind == DenseWeights::FLOAT16) gemm_float(x, w.weight.ptr, w.bias.ptr, residual, act, m, w.n, w.k, y, dtype, st);
  else dense_awq(x, awq_view(w), w.bias.ptr, residual, act, m, y, awq_scratch, st);
}

// =============================================================================================
// LlamaDecoder
// =============================================================================================
// Geometry and attributes of a TransformerDecoderSpec model directory (host only: no device is touched), with the checks
// for what this engine serves.  Attributes: models/model.h get_attribute_with_default; attention_layer.cc:112-142.
ModelConfig parse_model_config(const ModelFile& f) {
  ModelConfig mc;
  if (f.spec_name != "TransformerDecoderSpec")
    throw std::invalid_argument("ct2b200 serves TransformerDecoderSpec models; got " + f.spec_name);
  // --- configuration (attributes: models/model.h get_attribute_with_default; attention_layer.cc:112-142) ---
  while (f.find("decoder/layer_" + std::to_string(mc.num_layers) + "/self_attention/linear_0/weight")) ++mc.num_layers;
  CT2_REQUIRE(mc.num_layers > 0, "model has no decoder layers");
  const std::string a0 = "decoder/layer_0/self_attention/";
  mc.num_heads = static_cast<int>(f.get("decoder/num_heads").scalar());
  mc.num_heads_kv = static_cast<int>(f.attribute(a0 + "num_heads_kv", mc.num_heads));
  const HostVariable& emb = f.get("decoder/embeddings/weight");
  mc.vocab = emb.shape[0];
  mc.d_model = emb.shape[1];
  mc.head_dim = static_cast<int>(f.attribute(a0 + "head_dim", static_cast<double>(mc.d_model / mc.num_heads)));
  mc.eps = static_cast<float>(f.config_number("layer_norm_epsilon", 1e-6));
  mc.rotary_base = static_cast<float>(f.attribute(a0 + "rotary_base", 10000.0));
  mc.rotary_interleave = f.attribute(a0 + "rotary_interleave", 1.0) != 0.0;
  mc.rotary_scaling_type = static_cast<int>(f.attribute(a0 + "rotary_scaling_type", -1.0));
  mc.rotary_scaling_factor = static_cast<float>(f.attribute(a0 + "rotary_scaling_factor", 1.0));
  mc.rotary_low_freq = static_cast<float>(f.attribute(a0 + "rotary_low_freq_factor", 1.0));
  mc.rotary_high_freq = static_cast<float>(f.attribute(a0 + "rotary_high_freq_factor", 4.0));
  mc.original_max_positions = static_cast<int>(f.attribute(a0 + "original_max_position_embeddings", 0.0));
  mc.activation = static_cast<int>(f.attribute("decoder/activation", 0.0));
  CT2_REQUIRE(f.attribute("decoder/pre_norm", 1.0) != 0.0, "only pre-norm decoders are supported");
  CT2_REQUIRE(f.find(a0 + "rotary_dim") != nullptr, "only rotary-position decoders are supported");
  CT2_REQUIRE(f.attribute(a0 + "rotary_dim", 0.0) == 0.0 ||
                  f.attribute(a0 + "rotary_dim", 0.0) == mc.head_dim, "partial rotary_dim is not supported");
  CT2_REQUIRE(f.find("decoder/layer_0/ffn/linear_0_noact/weight") != nullptr, "only gated FFN (ffn_glu) is supported");
  CT2_REQUIRE(f.find("decoder/layer_0/self_attention/layer_norm/beta") == nullptr, "only RMSNorm decoders are supported");
  CT2_REQUIRE(mc.rotary_scaling_type != 1, "Su rotary scaling is not supported");
  // Features of TransformerDecoderSpec the reference honours and this engine does not implement: refuse the model instead
  // of silently computing something else (transformer.cc:380-400, 475-530; attention_layer.cc:112-142; common.cc:448).
  {
    // scale_embeddings: absent or a true int8 flag => embeddings * sqrt(d_model); a float => that factor (transformer.cc:385-396)
    const HostVariable* se = f.find("decoder/scale_embeddings");
    if (!se) se = f.find("decoder/embeddings/multiply_by_sqrt_depth");
    CT2_REQUIRE(se != nullptr, "decoder/scale_embeddings is absent: the reference would scale the embeddings by sqrt(d_model), "
                               "which this engine does not implement");
    CT2_REQUIRE((se->type_id == 1 && se->scalar() == 0.0) || (se->type_id != 1 && se->scalar() == 1.0),
                "scaled embeddings (decoder/scale_embeddings) are not supported");
    auto flag_off = [&](const std::string& name, const char* what) {
      if (f.attribute(name, 0.0) != 0.0) throw std::invalid_argument(std::string(what) + " (" + name + ") is not supported");
    };
    auto absent = [&](const std::string& name, const char* what) {
      if (f.find(name)) throw std::invalid_argument(std::string(what) + " (" + name + ") is not supported");
    };
    flag_off("decoder/alibi", "ALiBi positions");
    flag_off("decoder/sliding_window", "sliding-window attention");
    flag_off(a0 + "sliding_window", "sliding-window attention");
    flag_off(a0 + "multi_query", "the multi_query attention flag (use num_heads_kv)");
    flag_off("decoder/final_logit_softcapping", "final logit soft-capping");
    absent("decoder/scale_outputs", "scaled outputs");
    absent("decoder/layernorm_embedding/gamma", "layernorm_embedding");
    absent("decoder/project_in/weight", "project_in");
    absent("decoder/project_out/weight", "project_out");
    absent("decoder/position_encodings/encodings", "learned / sinusoidal position encodings");
    CT2_REQUIRE(f.attribute("decoder/layer_0/layer_scalar", 1.0) == 1.0, "layer_scalar is not supported");
    const double qs = f.attribute(a0 + "queries_scale", 0.0);
    CT2_REQUIRE(qs == 0.0 || std::fabs(qs - 1.0 / std::sqrt(static_cast<double>(mc.head_dim))) < 1e-6,
                "a queries_scale other than 1/sqrt(head_dim) is not supported");
    for (int l = 0; l < mc.num_layers; ++l) {
      const std::string p = "decoder/layer_" + std::to_string(l) + "/";
      absent(p + "self_attention/q_norm/gamma", "q_norm");
      absent(p + "self_attention/k_norm/gamma", "k_norm");
      absent(p + "self_attention/relative_position_keys", "relative positions");
      absent(p + "self_attention/relative_attention_bias", "relative attention bias");
      absent(p + "attention/linear_0/weight", "cross attention (encoder-decoder models)");
      for (const char* n : {"input_layer_norm", "post_attention_layer_norm", "pre_feedforward_layer_norm",
                            "post_feedforward_layer_norm", "shared_layer_norm"})
        absent(p + n + "/gamma", "an extra layer norm");
      flag_off(p + "self_attention/layer_norm/layer_norm_use_residual", "layer_norm_use_residual (1 + gamma)");
      flag_off(p + "ffn/layer_norm/layer_norm_use_residual", "layer_norm_use_residual (1 + gamma)");
    }
    flag_off("decoder/layer_norm/layer_norm_use_residual", "layer_norm_use_residual (1 + gamma)");
  }
  {
    // output features of the gate projection: rows of an int8 / float weight, columns x 8 of an AWQ_GEMM-packed one
    // (qweight [K, N/8]), rows of an AWQ_GEMV-packed one (qweight [N, K/8])
    const HostVariable& gw = f.get("decoder/layer_0/ffn/linear_0/weight");
    const bool awq = gw.type_id == 3 && f.find("decoder/layer_0/ffn/linear_0/weight_zero");
    mc.ffn_dim = (awq && static_cast<int>(f.config_number("quantization_type", 0)) == 1) ? gw.shape[1] * 8 : gw.shape[0];
  }
  {
    const HostVariable& qkv = f.get("decoder/layer_0/self_attention/linear_0/weight");
    const bool awq = qkv.type_id == 3 && f.find("decoder/layer_0/self_attention/linear_0/weight_zero");
    mc.weights = qkv.type_id == 1 ? "int8" : awq ? (static_cast<int>(f.config_number("quantization_type", 0)) == 1 ? "awq_gemm" : "awq_gemv")
               : qkv.type_id == 4 ? "float16" : qkv.type_id == 5 ? "bfloat16" : qkv.type_id == 0 ? "float32" : "unsupported";
  }
  {
    const HostVariable* g = f.find("decoder/layer_norm/gamma");
    mc.float_type = !g ? "float32" : g->type_id == 4 ? "float16" : g->type_id == 5 ? "bfloat16" : "float32";
  }
  return mc;
}

LlamaDecoder::LlamaDecoder(const ModelFile& f, const ct2b200_generator_config& cfg) : gpu_(cfg.device) {
  dtype_ = cfg.compute_type;
  gemm_impl_ = cfg.gemm_impl;
  weight_type_ = cfg.weight_type;
  CT2_REQUIRE(weight_type_ >= 0 && weight_type_ <= 2, "weight_type must be a ct2b200_weight_type");
  max_batch_ = std::max<int64_t>(1, cfg.max_batch);
  max_len_ = std::max<int64_t>(16, cfg.max_length);
  tp_.world = std::max(1, cfg.tp_size);
  tp_.rank = cfg.tp_rank;
  CT2_REQUIRE(tp_.world <= 8 && tp_.rank >= 0 && tp_.rank < tp_.world, "tensor parallel: rank/size out of range (size <= 8)");

  mc_ = parse_model_config(f);
  CT2_REQUIRE(mc_.num_heads % tp_.world == 0 && mc_.num_heads_kv % tp_.world == 0 && mc_.ffn_dim % tp_.world == 0,
              "tensor parallel: heads, kv heads and ffn width must be divisible by the number of ranks");
  heads_ = mc_.num_heads / tp_.world;
  heads_kv_ = mc_.num_heads_kv / tp_.world;
  ffn_ = mc_.ffn_dim / tp_.world;

  // --- weights ---
  DenseLoad opt{dtype_, weight_type_, stream(), Shard::REPLICATED, mc_.num_heads, mc_.num_heads_kv, mc_.head_dim, tp_.rank,
                tp_.world, /*awq=*/true};
  auto dense = [&](const std::string& prefix, DenseWeights& w, Shard shard) {
    opt.shard = shard;
    mc_.weight_bytes += load_dense(f, prefix, opt, w);
  };
  auto gamma = [&](const std::string& name, DeviceBuffer& g) { mc_.weight_bytes += upload_as(g, f.get(name), dtype_); };
  dense("decoder/embeddings", embeddings_, Shard::REPLICATED);
  mc_.embeddings_int8 = embeddings_.kind == DenseWeights::INT8;
  dense("decoder/projection", projection_, Shard::REPLICATED);
  gamma("decoder/layer_norm/gamma", final_gamma_);
  layers_.resize(mc_.num_layers);
  for (int l = 0; l < mc_.num_layers; ++l) {
    const std::string p = "decoder/layer_" + std::to_string(l) + "/";
    LayerWeights& lw = layers_[l];
    gamma(p + "self_attention/layer_norm/gamma", lw.attn_gamma);
    gamma(p + "ffn/layer_norm/gamma", lw.ffn_gamma);
    dense(p + "self_attention/linear_0", lw.qkv, Shard::QKV_ROWS);
    dense(p + "self_attention/linear_1", lw.out, Shard::COLS);
    dense(p + "ffn/linear_0", lw.gate, Shard::ROWS);
    dense(p + "ffn/linear_0_noact", lw.up, Shard::ROWS);
    dense(p + "ffn/linear_1", lw.down, Shard::COLS);
  }

  // --- rotary tables, fp32 (RotaryEmbeddings::initialize, attention_layer.cc:252-343) ---
  {
    const int D = mc_.head_dim;
    std::vector<float> inv(D / 2);
    for (int i = 0; i < D / 2; ++i) inv[i] = 1.f / std::pow(mc_.rotary_base, static_cast<float>(i * 2) / static_cast<float>(D));
    if (mc_.rotary_scaling_type == 2) {   // Llama3
      const float old_len = static_cast<float>(mc_.original_max_positions);
      const float low_wl = old_len / mc_.rotary_low_freq, high_wl = old_len / mc_.rotary_high_freq;
      std::vector<float> nf = inv;
      for (int i = 0; i < D / 2; ++i) {
        const float wl = 2.0f * static_cast<float>(M_PI) / inv[i];
        if (wl < high_wl) {
        } else if (wl > low_wl) nf[i] = inv[i] / mc_.rotary_scaling_factor;
        else {
          const float smooth = (old_len / wl - mc_.rotary_low_freq) / (mc_.rotary_high_freq - mc_.rotary_low_freq);
          nf[i] = (1 - smooth) * inv[i] / mc_.rotary_scaling_factor + smooth * inv[i];
        }
      }
      inv = nf;
    }
    std::vector<float> sn(max_len_ * D), cs(max_len_ * D);
    for (int64_t t = 0; t < max_len_; ++t) {
      const float tt = mc_.rotary_scaling_type == 0 ? static_cast<float>(t) / mc_.rotary_scaling_factor : static_cast<float>(t);
      for (int i = 0; i < D; ++i) {
        const int fi = mc_.rotary_interleave ? i / 2 : i % (D / 2);
        const float ang = tt * inv[fi];
        sn[t * D + i] = std::sin(ang);
        cs[t * D + i] = std::cos(ang);
      }
    }
    upload(sin_, sn.data(), sn.size() * 4);
    upload(cos_, cs.data(), cs.size() * 4);
  }

  // --- KV arena + activations ---
  const size_t es = dtype_size(dtype_);
  const size_t cache_bytes = static_cast<size_t>(max_batch_) * heads_kv_ * max_len_ * mc_.head_dim * es;
  k_cache_.resize(mc_.num_layers);
  v_cache_.resize(mc_.num_layers);
  for (int l = 0; l < mc_.num_layers; ++l) {
    k_cache_[l].alloc(cache_bytes);
    v_cache_[l].alloc(cache_bytes);
    // the TMA-staged attention reads whole 64-key boxes: keys past the end are masked, but must be finite
    CT2_CUDA_CHECK(cudaMemsetAsync(k_cache_[l].ptr, 0, cache_bytes, stream()));
    CT2_CUDA_CHECK(cudaMemsetAsync(v_cache_[l].ptr, 0, cache_bytes, stream()));
  }
  chunk_rows_ = std::max<int64_t>(max_batch_, std::min<int64_t>(8192, max_batch_ * max_len_));
  const int64_t R = chunk_rows_;
  const int64_t qkv_w = static_cast<int64_t>(heads_ + 2 * heads_kv_) * mc_.head_dim;
  x_.alloc(R * mc_.d_model * es);
  xq_.alloc(R * std::max(mc_.d_model, mc_.ffn_dim));
  xs_.alloc(R * sizeof(float));
  qkv_.alloc(R * qkv_w * es);
  attn_.alloc(R * heads_ * mc_.head_dim * es);
  h_.alloc(R * ffn_ * es);
  if (layers_[0].qkv.kind != DenseWeights::INT8 || projection_.kind != DenseWeights::INT8) {
    xn_.alloc(R * mc_.d_model * es);
    scratch_mn_.alloc(R * mc_.ffn_dim * es);
    if (layers_[0].qkv.kind != DenseWeights::FLOAT16)
      scratch_nk_.alloc(static_cast<size_t>(std::max(mc_.ffn_dim, mc_.d_model)) * std::max<int64_t>(mc_.ffn_dim, qkv_w) * 2);
  }
  logits_.alloc(max_batch_ * mc_.vocab * es);
  gathered_.alloc(max_batch_ * mc_.d_model * es);
  attn_splits_ = attention_decode_splits(max_batch_, heads_kv_, max_len_, gpu_.sm_count);
  attn_ws_.alloc(attention_decode_workspace_bytes(max_batch_, heads_, mc_.head_dim, std::max(attn_splits_, 80)));
  CT2_CUDA_CHECK(cudaMemset(attn_ws_.ptr, 0, attn_ws_.bytes));
  CT2_CUDA_CHECK(cudaDeviceSynchronize());   // legacy-stream memset vs the engine's non-blocking stream
  if (tp_.world > 1) {
    // exchange buffer of this rank: [flags 2x8 u32 | pad to 256] [amax words 2 x 8 x R] [partials 2 x R x d_model]
    tp_.flags_off = 0;
    tp_.amax_off = 256;
    const size_t amax_bytes = static_cast<size_t>(2) * 8 * R * sizeof(unsigned long long);
    const size_t part_bytes = ((static_cast<size_t>(R) * mc_.d_model * es + 255) / 256) * 256;
    tp_.part_off[0] = tp_.amax_off + ((amax_bytes + 255) / 256) * 256;
    tp_.part_off[1] = tp_.part_off[0] + part_bytes;
    tp_.exchange.alloc(tp_.part_off[1] + part_bytes);
    CT2_CUDA_CHECK(cudaMemset(tp_.exchange.ptr, 0, tp_.exchange.bytes));
    CT2_CUDA_CHECK(cudaDeviceSynchronize());   // legacy-stream memset vs the engine's non-blocking stream
    tp_.tick.alloc(256);
    CT2_CUDA_CHECK(cudaMemset(tp_.tick.ptr, 0, 256));
    CT2_CUDA_CHECK(cudaDeviceSynchronize());   // legacy-stream memset vs the engine's non-blocking stream
  }
  CT2_CUDA_CHECK(cudaDeviceSynchronize());
}

LlamaDecoder::~LlamaDecoder() {
  cudaSetDevice(gpu_.device);
  // the peer exchange buffers mapped by tp_connect are unmapped once nothing in flight reads them, before gpu_ goes away
  cudaStreamSynchronize(stream());
  for (int r = 0; r < tp_.world; ++r)
    if (tp_.connected && r != tp_.rank && tp_.peer[r]) cudaIpcCloseMemHandle(tp_.peer[r]);
}

void LlamaDecoder::dense(const DenseWeights& w, const int8_t* xq, const float* xs, const void* x_float, int64_t m,
                         const void* residual, int act, void* y) {
  dense_forward(w, xq, xs, x_float, m, residual, act, y, 0, dtype_, gemm_impl_, scratch_nk_.ptr, stream());
}

// [RMSNorm +] Quantize + Dense: the row kernel, then the GEMM under programmatic dependent launch.
void LlamaDecoder::dense_from_rows(const DenseWeights& w, const void* x_rows, const void* gamma, int64_t cols, int64_t m,
                                   const void* residual, int act, void* y) {
  rows_to_int8(x_rows, gamma, mc_.eps, m, cols, dtype_, xq_.as<int8_t>(), xs_.as<float>(), stream());
  dense(w, xq_.as<int8_t>(), xs_.as<float>(), nullptr, m, residual, act, y);
}

void LlamaDecoder::glu_from_rows(const DenseWeights& gate, const DenseWeights& up, const void* x_rows, const void* gamma,
                                 int64_t m, void* h) {
  GluEpilogue g{xs_.as<float>(), gate.scale.as<float>(), up.scale.as<float>(), h, mc_.activation, gate.n};
  rows_to_int8(x_rows, gamma, mc_.eps, m, gate.k, dtype_, xq_.as<int8_t>(), xs_.as<float>(), stream());
  gemm_s8_glu(xq_.as<int8_t>(), gate.weight.as<int8_t>(), up.weight.as<int8_t>(), m, gate.n, gate.k, g, dtype_, gemm_impl_,
              stream());
}

void LlamaDecoder::layers_forward(int64_t rows, int64_t batch, int64_t time, int64_t offset, const int32_t* lens_d) {
  if (tp_.world > 1) {
    layers_forward_tp(rows, batch, time, offset, lens_d);
    return;
  }
  const int H = mc_.num_heads, Hkv = mc_.num_heads_kv, D = mc_.head_dim;
  const float scale = 1.f / std::sqrt(static_cast<float>(D));
  const bool int8 = layers_[0].qkv.kind == DenseWeights::INT8;
  auto attention = [&](int l) {
    if (lens_d) {
      launch_attention_decode(qkv_.ptr, k_cache_[l].ptr, v_cache_[l].ptr, sin_.as<float>(), cos_.as<float>(), lens_d,
                              batch, H, Hkv, D, max_len_, mc_.rotary_interleave, scale, attn_.ptr, attn_ws_.ptr,
                              attn_ws_.bytes, attn_splits_, dtype_, stream());
    } else {
      launch_rope_append(qkv_.ptr, k_cache_[l].ptr, v_cache_[l].ptr, sin_.as<float>(), cos_.as<float>(), nullptr,
                         batch, time, offset, H, Hkv, D, max_len_, mc_.rotary_interleave, dtype_, stream());
      launch_attention_prefill(qkv_.ptr, k_cache_[l].ptr, v_cache_[l].ptr, nullptr, batch, time, offset, H, Hkv, D,
                               max_len_, scale, attn_.ptr, dtype_, stream());
    }
  };
  if (!int8) {
    // float16/bfloat16 weights (Dense float arm, common.cc:440) and AWQ-INT4 (common.cc:402-438): activations stay in T
    for (int l = 0; l < mc_.num_layers; ++l) {
      LayerWeights& lw = layers_[l];
      launch_rms_norm(lw.attn_gamma.ptr, x_.ptr, rows, mc_.d_model, mc_.eps, false, xn_.ptr, nullptr, nullptr, dtype_, stream());
      dense(lw.qkv, nullptr, nullptr, xn_.ptr, rows, nullptr, -1, qkv_.ptr);
      attention(l);
      dense(lw.out, nullptr, nullptr, attn_.ptr, rows, x_.ptr, -1, x_.ptr);
      launch_rms_norm(lw.ffn_gamma.ptr, x_.ptr, rows, mc_.d_model, mc_.eps, false, xn_.ptr, nullptr, nullptr, dtype_, stream());
      if (lw.gate.kind == DenseWeights::FLOAT16) {
        dense(lw.gate, nullptr, nullptr, xn_.ptr, rows, nullptr, mc_.activation, h_.ptr);
        dense(lw.up, nullptr, nullptr, xn_.ptr, rows, nullptr, -1, scratch_mn_.ptr);
        launch_mul_inplace(h_.ptr, scratch_mn_.ptr, rows * mc_.ffn_dim, dtype_, stream());
      } else {
        dense_awq_glu(xn_.ptr, awq_view(lw.gate), awq_view(lw.up), mc_.activation, rows, h_.ptr, scratch_nk_.ptr,
                      scratch_mn_.ptr, stream());
      }
      dense(lw.down, nullptr, nullptr, h_.ptr, rows, x_.ptr, -1, x_.ptr);
    }
    return;
  }
  // Per layer: RMSNorm + Quantize, QKV Dense, attention, Quantize, out Dense (+ residual), RMSNorm + Quantize, gate/up Dense with
  // SwiGLU, Quantize, down Dense (+ residual): 9 launches, every one with programmatic dependent launch.
  for (int l = 0; l < mc_.num_layers; ++l) {
    LayerWeights& lw = layers_[l];
    // --- self attention (attention.cc:442-615) ---
    dense_from_rows(lw.qkv, x_.ptr, lw.attn_gamma.ptr, mc_.d_model, rows, nullptr, -1, qkv_.ptr);
    attention(l);
    dense_from_rows(lw.out, attn_.ptr, nullptr, static_cast<int64_t>(H) * D, rows, x_.ptr, -1, x_.ptr);
    // --- feed forward (transformer.cc:21-51) ---
    glu_from_rows(lw.gate, lw.up, x_.ptr, lw.ffn_gamma.ptr, rows, h_.ptr);
    dense_from_rows(lw.down, h_.ptr, nullptr, mc_.ffn_dim, rows, x_.ptr, -1, x_.ptr);
  }
}

// Tensor-parallel layer stack (one process per GPU).  Per layer, rank r computes its heads / FFN columns; the two
// all-reduces of the reference (attention.cc:608-612, transformer.cc:45-48) are fused into the next kernel on the
// residual stream and the activation all-gather before a row-parallel INT8 Dense (common.cc:360-387) into the
// quantization kernel (kernels/tp_rows.cu).  Sync point indices of a pass: 4l amax(attention out), 4l+1 sum(out-proj),
// 4l+2 amax(ffn hidden), 4l+3 sum(down-proj).
void LlamaDecoder::layers_forward_tp(int64_t rows, int64_t batch, int64_t time, int64_t offset, const int32_t* lens_d) {
  CT2_REQUIRE(tp_.connected, "tensor parallel: call ct2b200_generator_tp_connect before running the model");
  const int H = heads_, Hkv = heads_kv_, D = mc_.head_dim;
  const float scale = 1.f / std::sqrt(static_cast<float>(D));
  const bool int8 = layers_[0].qkv.kind == DenseWeights::INT8;
  const TpLink& tp = tp_.link;
  void* part[2] = {static_cast<uint8_t*>(tp_.exchange.ptr) + tp_.part_off[0],
                   static_cast<uint8_t*>(tp_.exchange.ptr) + tp_.part_off[1]};
  launch_tp_tick(tp_.tick.as<uint32_t>(), stream());
  auto attention = [&](int l) {
    if (lens_d) {
      launch_attention_decode(qkv_.ptr, k_cache_[l].ptr, v_cache_[l].ptr, sin_.as<float>(), cos_.as<float>(), lens_d,
                              batch, H, Hkv, D, max_len_, mc_.rotary_interleave, scale, attn_.ptr, attn_ws_.ptr,
                              attn_ws_.bytes, attn_splits_, dtype_, stream());
    } else {
      launch_rope_append(qkv_.ptr, k_cache_[l].ptr, v_cache_[l].ptr, sin_.as<float>(), cos_.as<float>(), nullptr,
                         batch, time, offset, H, Hkv, D, max_len_, mc_.rotary_interleave, dtype_, stream());
      launch_attention_prefill(qkv_.ptr, k_cache_[l].ptr, v_cache_[l].ptr, nullptr, batch, time, offset, H, Hkv, D,
                               max_len_, scale, attn_.ptr, dtype_, stream());
    }
  };
  for (int l = 0; l < mc_.num_layers; ++l) {
    LayerWeights& lw = layers_[l];
    if (int8) {
      if (l == 0)
        launch_rms_norm(lw.attn_gamma.ptr, x_.ptr, rows, mc_.d_model, mc_.eps, false, nullptr, xq_.as<int8_t>(),
                        xs_.as<float>(), dtype_, stream());
      else
        launch_tp_reduce_norm_quantize(tp, 1, 4 * (l - 1) + 3, x_.ptr, lw.attn_gamma.ptr, rows, mc_.d_model, mc_.eps,
                                       xq_.as<int8_t>(), xs_.as<float>(), dtype_, stream());
      dense(lw.qkv, xq_.as<int8_t>(), xs_.as<float>(), nullptr, rows, nullptr, -1, qkv_.ptr);
      attention(l);
      launch_tp_quantize_rows(tp, 0, 4 * l, attn_.ptr, rows, static_cast<int64_t>(H) * D, xq_.as<int8_t>(),
                              xs_.as<float>(), dtype_, stream());
      dense(lw.out, xq_.as<int8_t>(), xs_.as<float>(), nullptr, rows, nullptr, -1, part[0]);
      launch_tp_reduce_norm_quantize(tp, 0, 4 * l + 1, x_.ptr, lw.ffn_gamma.ptr, rows, mc_.d_model, mc_.eps,
                                     xq_.as<int8_t>(), xs_.as<float>(), dtype_, stream());
      GluEpilogue g{xs_.as<float>(), lw.gate.scale.as<float>(), lw.up.scale.as<float>(), h_.ptr, mc_.activation, lw.gate.n};
      gemm_s8_glu(xq_.as<int8_t>(), lw.gate.weight.as<int8_t>(), lw.up.weight.as<int8_t>(), rows, lw.gate.n, lw.gate.k, g,
                  dtype_, gemm_impl_, stream());
      launch_tp_quantize_rows(tp, 1, 4 * l + 2, h_.ptr, rows, ffn_, xq_.as<int8_t>(), xs_.as<float>(), dtype_, stream());
      dense(lw.down, xq_.as<int8_t>(), xs_.as<float>(), nullptr, rows, nullptr, -1, part[1]);
    } else {
      if (l == 0)
        launch_rms_norm(lw.attn_gamma.ptr, x_.ptr, rows, mc_.d_model, mc_.eps, false, xn_.ptr, nullptr, nullptr, dtype_, stream());
      else
        launch_tp_reduce_norm(tp, 1, 4 * (l - 1) + 3, x_.ptr, lw.attn_gamma.ptr, rows, mc_.d_model, mc_.eps, xn_.ptr, dtype_, stream());
      dense(lw.qkv, nullptr, nullptr, xn_.ptr, rows, nullptr, -1, qkv_.ptr);
      attention(l);
      dense(lw.out, nullptr, nullptr, attn_.ptr, rows, nullptr, -1, part[0]);
      launch_tp_reduce_norm(tp, 0, 4 * l + 1, x_.ptr, lw.ffn_gamma.ptr, rows, mc_.d_model, mc_.eps, xn_.ptr, dtype_, stream());
      dense(lw.gate, nullptr, nullptr, xn_.ptr, rows, nullptr, mc_.activation, h_.ptr);
      dense(lw.up, nullptr, nullptr, xn_.ptr, rows, nullptr, -1, scratch_mn_.ptr);
      launch_mul_inplace(h_.ptr, scratch_mn_.ptr, rows * ffn_, dtype_, stream());
      dense(lw.down, nullptr, nullptr, h_.ptr, rows, nullptr, -1, part[1]);
    }
  }
  // the residual stream is complete once the last down-proj partials are summed in
  launch_tp_reduce(tp, 1, 4 * (mc_.num_layers - 1) + 3, x_.ptr, rows, mc_.d_model, dtype_, stream());
}

void LlamaDecoder::tp_handle(void* handle64) const {
  CT2_REQUIRE(tp_.world > 1 && tp_.exchange.ptr, "tensor parallel is not enabled for this generator (tp_size == 1)");
  static_assert(sizeof(cudaIpcMemHandle_t) == 64, "cudaIpcMemHandle_t is 64 bytes");
  cudaIpcMemHandle_t h;
  CT2_CUDA_CHECK(cudaIpcGetMemHandle(&h, tp_.exchange.ptr));
  std::memcpy(handle64, &h, sizeof(h));
}

void LlamaDecoder::tp_connect(const void* handles, int count) {
  CT2_REQUIRE(tp_.world > 1, "tensor parallel is not enabled for this generator (tp_size == 1)");
  CT2_REQUIRE(count == tp_.world, "tp_connect: one handle per rank is required");
  CT2_CUDA_CHECK(cudaSetDevice(gpu_.device));
  for (int r = 0; r < tp_.world; ++r) {
    if (r == tp_.rank) {
      tp_.peer[r] = tp_.exchange.ptr;
      continue;
    }
    cudaIpcMemHandle_t h;
    std::memcpy(&h, static_cast<const uint8_t*>(handles) + static_cast<size_t>(r) * sizeof(h), sizeof(h));
    CT2_CUDA_CHECK(cudaIpcOpenMemHandle(&tp_.peer[r], h, cudaIpcMemLazyEnablePeerAccess));
  }
  TpLink& k = tp_.link;
  k.rank = tp_.rank;
  k.world = tp_.world;
  k.tick = tp_.tick.as<uint32_t>();
  k.amax_rows = chunk_rows_;
  k.flags_local = reinterpret_cast<uint32_t*>(static_cast<uint8_t*>(tp_.exchange.ptr) + tp_.flags_off);
  k.amax_local = reinterpret_cast<unsigned long long*>(static_cast<uint8_t*>(tp_.exchange.ptr) + tp_.amax_off);
  for (int r = 0; r < tp_.world; ++r) {
    uint8_t* base = static_cast<uint8_t*>(tp_.peer[r]);
    k.flags_peer[r] = reinterpret_cast<uint32_t*>(base + tp_.flags_off);
    k.amax_peer[r] = reinterpret_cast<unsigned long long*>(base + tp_.amax_off);
    k.parts[0][r] = base + tp_.part_off[0];
    k.parts[1][r] = base + tp_.part_off[1];
  }
  tp_.connected = true;
}

// layers::Embeddings::operator() (common.cc:64-81)
void LlamaDecoder::embed(const int32_t* ids_d, int64_t rows) {
  if (embeddings_.kind == DenseWeights::INT8)
    launch_embedding_s8(embeddings_.weight.as<int8_t>(), embeddings_.scale.as<float>(), ids_d, rows, mc_.d_model, x_.ptr,
                        dtype_, stream());
  else
    launch_gather_rows(embeddings_.weight.ptr, ids_d, rows, mc_.d_model * dtype_size(dtype_), x_.ptr, stream());
}

void LlamaDecoder::project(const void* x_rows, int64_t rows, void* logits_out) {
  if (projection_.kind == DenseWeights::INT8) {
    launch_rms_norm(final_gamma_.ptr, x_rows, rows, mc_.d_model, mc_.eps, false, nullptr, xq_.as<int8_t>(),
                    xs_.as<float>(), dtype_, stream());
    dense(projection_, xq_.as<int8_t>(), xs_.as<float>(), nullptr, rows, nullptr, -1, logits_out);
  } else {
    launch_rms_norm(final_gamma_.ptr, x_rows, rows, mc_.d_model, mc_.eps, false, xn_.ptr, nullptr, nullptr, dtype_, stream());
    dense(projection_, nullptr, nullptr, xn_.ptr, rows, nullptr, -1, logits_out);
  }
}

void LlamaDecoder::forward_prefill(const int32_t* ids_d, int64_t batch, int64_t time, int64_t offset,
                                   void* logits_out_d, const int32_t* logits_rows_d, int64_t num_logit_rows) {
  const int64_t rows = batch * time;
  CT2_REQUIRE(rows <= chunk_rows_, "forward_prefill: too many rows for the activation arena");
  CT2_REQUIRE(batch <= max_batch_ && offset + time <= max_len_, "forward_prefill: batch/length exceeds the KV arena");
  embed(ids_d, rows);
  layers_forward(rows, batch, time, offset, nullptr);
  if (logits_out_d && num_logit_rows > 0) {
    if (logits_rows_d) {
      CT2_REQUIRE(num_logit_rows <= max_batch_, "too many logit rows");
      launch_gather_rows(x_.ptr, logits_rows_d, num_logit_rows, mc_.d_model * dtype_size(dtype_), gathered_.ptr, stream());
      project(gathered_.ptr, num_logit_rows, logits_out_d);
    } else {
      project(x_.ptr, num_logit_rows, logits_out_d);
    }
  }
}

void LlamaDecoder::project_rows(const int32_t* rows_d, int64_t n, void* logits_out_d) {
  CT2_REQUIRE(n <= max_batch_, "project_rows: too many rows");
  launch_gather_rows(x_.ptr, rows_d, n, mc_.d_model * dtype_size(dtype_), gathered_.ptr, stream());
  project(gathered_.ptr, n, logits_out_d);
}

void LlamaDecoder::gather_hidden(const int32_t* rows_d, int64_t n, void* out_d) {
  launch_gather_rows(x_.ptr, rows_d, n, mc_.d_model * dtype_size(dtype_), out_d, stream());
}

void LlamaDecoder::project_hidden(const void* x_rows_d, int64_t rows, void* logits_out_d) {
  CT2_REQUIRE(rows <= chunk_rows_, "project_hidden: too many rows for the activation arena");
  project(x_rows_d, rows, logits_out_d);
}

void LlamaDecoder::reorder_cache(const int32_t* parent_d, int beam, int64_t rows, int64_t positions) {
  CT2_REQUIRE(tp_.world == 1, "beam search does not run tensor parallel");
  CT2_REQUIRE(rows <= max_batch_ && positions <= max_len_, "reorder_cache: exceeds the KV arena");
  if (k_alt_.empty()) {
    k_alt_.resize(mc_.num_layers);
    v_alt_.resize(mc_.num_layers);
    for (int l = 0; l < mc_.num_layers; ++l) {
      k_alt_[l].alloc(k_cache_[l].bytes);
      v_alt_[l].alloc(v_cache_[l].bytes);
      // whole 64-key boxes are staged by the attention kernels: positions past the end must hold finite values
      CT2_CUDA_CHECK(cudaMemsetAsync(k_alt_[l].ptr, 0, k_alt_[l].bytes, stream()));
      CT2_CUDA_CHECK(cudaMemsetAsync(v_alt_[l].ptr, 0, v_alt_[l].bytes, stream()));
    }
  }
  for (int l = 0; l < mc_.num_layers; ++l) {
    launch_kv_gather(k_cache_[l].ptr, v_cache_[l].ptr, k_alt_[l].ptr, v_alt_[l].ptr, parent_d, beam, rows, heads_kv_, max_len_,
                     mc_.head_dim, positions, dtype_, stream());
    std::swap(k_cache_[l], k_alt_[l]);
    std::swap(v_cache_[l], v_alt_[l]);
  }
  cache_swapped_ = !cache_swapped_;
}

void LlamaDecoder::restore_cache_orientation() {
  if (!cache_swapped_) return;
  for (int l = 0; l < mc_.num_layers; ++l) {
    std::swap(k_cache_[l], k_alt_[l]);
    std::swap(v_cache_[l], v_alt_[l]);
  }
  cache_swapped_ = false;
}

void LlamaDecoder::forward_step(const int32_t* ids_d, const int32_t* lens_d, int64_t batch, void* logits_out_d) {
  CT2_REQUIRE(batch <= max_batch_, "forward_step: batch exceeds the KV arena");
  embed(ids_d, batch);
  layers_forward(batch, batch, 1, 0, lens_d);
  project(x_.ptr, batch, logits_out_d);
}

// =============================================================================================
// Generator
// =============================================================================================
Generator::Generator(const std::string& model_dir, const ct2b200_generator_config& cfg) : cfg_(cfg) {
  ModelFile file(model_dir);
  decoder_ = std::make_unique<LlamaDecoder>(file, cfg);
  const int64_t B = decoder_->max_batch(), L = decoder_->max_length();
  ids_d_.alloc(std::max<int64_t>(B, decoder_->prefill_chunk_rows()) * sizeof(int32_t));
  lens_d_.alloc(B * sizeof(int32_t));
  step_d_.alloc(8 * sizeof(int32_t));
  attn_lens_d_.alloc(B * sizeof(int32_t));
  finished_d_.alloc(B * sizeof(int32_t));
  forced_d_.alloc(B * L * sizeof(int32_t));
  out_d_.alloc(B * L * sizeof(int32_t));
  end_ids_d_.alloc(64 * sizeof(int32_t));
  sample_ws_.alloc((B * 97) * sizeof(int32_t));      // part_v [B*32] | part_i [B*32] | tickets [B] | part_s [B*32]
  scores_d_.alloc(B * L * sizeof(float));             // per-step log-probabilities (return_scores)
  row_start_d_.alloc(B * sizeof(int32_t));            // first loop step whose sample is a generated token, per row
  CT2_CUDA_CHECK(cudaMemset(row_start_d_.ptr, 0, row_start_d_.bytes));
  CT2_CUDA_CHECK(cudaMemset(sample_ws_.ptr, 0, sample_ws_.bytes));
  CT2_CUDA_CHECK(cudaDeviceSynchronize());   // legacy-stream memset vs the engine's non-blocking stream
  prompt_d_.alloc(B * L * sizeof(int32_t));
  host_pinned_elems_ = static_cast<size_t>(B) * (L + 2) + 256;   // prompt block | forced inputs | gen[4] | end ids[64] | row starts[B]
  CT2_CUDA_CHECK(cudaMallocHost(&host_pinned_, host_pinned_elems_ * sizeof(int32_t)));
}

Generator::~Generator() {
  if (host_pinned_) cudaFreeHost(host_pinned_);
  if (score_pinned_) cudaFreeHost(score_pinned_);
}

// prefill `time` tokens per row from position 0, in row chunks that fit the activation arena
void Generator::run_prefill(const int32_t* ids_d, int64_t batch, int64_t time,
                            const std::function<void(int64_t, int64_t)>& after_chunk) {
  LlamaDecoder& d = *decoder_;
  const int64_t tc_max = std::max<int64_t>(1, d.prefill_chunk_rows() / batch);
  for (int64_t t0 = 0; t0 < time; t0 += tc_max) {
    const int64_t tc = std::min(tc_max, time - t0);
    // gather the [batch, tc] slice of the [batch, time] id matrix into a dense block
    CT2_CUDA_CHECK(cudaMemcpy2DAsync(ids_d_.ptr, tc * sizeof(int32_t), ids_d + t0, time * sizeof(int32_t),
                                     tc * sizeof(int32_t), batch, cudaMemcpyDeviceToDevice, d.stream()));
    d.forward_prefill(ids_d_.as<int32_t>(), batch, tc, t0, nullptr, nullptr, 0);
    if (after_chunk) after_chunk(t0, tc);
  }
}

void Generator::launch_step(int64_t batch) {
  LlamaDecoder& d = *decoder_;
  d.forward_step(ids_d_.as<int32_t>(), attn_lens_d_.as<int32_t>(), batch, d.logits_buffer());
  launch_sample_greedy(d.logits_buffer(), batch, d.config().vocab, step_d_.as<int32_t>(), end_ids_d_.as<int32_t>(),
                       forced_d_.as<int32_t>(), ids_d_.as<int32_t>(), out_d_.as<int32_t>(), lens_d_.as<int32_t>(),
                       sample_ws_.as<float>(), sample_ws_.as<int32_t>() + d.max_batch() * 32,
                       sample_ws_.as<int32_t>() + d.max_batch() * 64, sample_ws_.as<float>() + d.max_batch() * 65,
                       want_scores_ ? scores_d_.as<float>() : nullptr, row_start_d_.as<int32_t>(), attn_lens_d_.as<int32_t>(),
                       finished_d_.as<int32_t>(), d.dtype(), d.stream());
}

void Generator::generate(const GenerationRequest& r, int32_t* out_ids, int32_t* out_lens, float* out_scores) {
  std::lock_guard<std::mutex> lock(mu_);      // one request at a time per generator (the reference queues them per replica)
  want_scores_ = r.return_scores && out_scores != nullptr;
  LlamaDecoder& d = *decoder_;
  cudaStream_t st = d.stream();
  const int64_t B = r.batch;
  CT2_REQUIRE(B > 0 && B <= d.max_batch(), "generate_batch: batch size exceeds max_batch");
  CT2_REQUIRE(r.end_ids.size() <= 64, "at most 64 end tokens");
  int64_t min_p = INT64_MAX, max_p = 0;
  for (int64_t b = 0; b < B; ++b) {
    CT2_REQUIRE(r.prompt_lens[b] >= 1, "generate_batch: every prompt needs at least one token (start token)");
    min_p = std::min<int64_t>(min_p, r.prompt_lens[b]);
    max_p = std::max<int64_t>(max_p, r.prompt_lens[b]);
  }
  CT2_REQUIRE(max_p + r.max_length <= d.max_length(), "generate_batch: prompt + max_length exceeds max_length of the KV arena");
  // language_model.cc:217-238: forward min_prompt_length-1 tokens at once, the rest goes through the loop
  const int64_t fwd = min_p - 1;
  const int64_t forced_steps = max_p - fwd;           // steps whose input is still a prompt token (>= 1)
  const int64_t total_steps = (max_p - min_p) + r.max_length;

  // host staging (pinned): prompt block [B, fwd], forced inputs [forced_steps, B], first ids
  int32_t* hp = host_pinned_;
  for (int64_t b = 0; b < B; ++b)
    for (int64_t t = 0; t < fwd; ++t) hp[b * fwd + t] = r.prompt_ids[b * r.max_prompt_len + t];
  int32_t* hforced = hp + B * fwd;
  for (int64_t s = 0; s < forced_steps; ++s)
    for (int64_t b = 0; b < B; ++b) {
      const int64_t t = fwd + s;
      hforced[s * B + b] = t < r.prompt_lens[b] ? r.prompt_ids[b * r.max_prompt_len + t] : -1;
    }
  int32_t* hgen = hforced + forced_steps * B;
  hgen[0] = static_cast<int32_t>(fwd);
  hgen[1] = 0;
  hgen[2] = static_cast<int32_t>(r.end_ids.size());
  hgen[3] = static_cast<int32_t>(forced_steps);
  // min_length counts GENERATED tokens per row: the kernel compares step - row_start[b] with it
  hgen[1] = static_cast<int32_t>(r.min_length);
  hgen[4] = static_cast<int32_t>(r.max_length);
  hgen[5] = hgen[6] = hgen[7] = 0;
  int32_t* hend = hgen + 8;
  for (size_t i = 0; i < r.end_ids.size(); ++i) hend[i] = r.end_ids[i];
  // step s consumes prompt token fwd + s; row b's first generated token is the sample of step prompt_len - 1 - fwd
  int32_t* hstart = hend + 64;
  for (int64_t b = 0; b < B; ++b) hstart[b] = static_cast<int32_t>(r.prompt_lens[b] - 1 - fwd);

  if (fwd > 0)
    CT2_CUDA_CHECK(cudaMemcpyAsync(prompt_d_.ptr, hp, B * fwd * sizeof(int32_t), cudaMemcpyHostToDevice, st));
  CT2_CUDA_CHECK(cudaMemcpyAsync(forced_d_.ptr, hforced, forced_steps * B * sizeof(int32_t), cudaMemcpyHostToDevice, st));
  CT2_CUDA_CHECK(cudaMemcpyAsync(step_d_.ptr, hgen, 8 * sizeof(int32_t), cudaMemcpyHostToDevice, st));
  if (!r.end_ids.empty())
    CT2_CUDA_CHECK(cudaMemcpyAsync(end_ids_d_.ptr, hend, r.end_ids.size() * sizeof(int32_t), cudaMemcpyHostToDevice, st));
  CT2_CUDA_CHECK(cudaMemcpyAsync(row_start_d_.ptr, hstart, B * sizeof(int32_t), cudaMemcpyHostToDevice, st));
  if (fwd > 0) run_prefill(prompt_d_.as<int32_t>(), B, fwd);
  // first decode input = forced[0] (the last common prompt token); positions = fwd
  CT2_CUDA_CHECK(cudaMemcpyAsync(ids_d_.ptr, forced_d_.ptr, B * sizeof(int32_t), cudaMemcpyDeviceToDevice, st));
  launch_fill_i32(lens_d_.as<int32_t>(), B, static_cast<int32_t>(fwd), st);
  launch_fill_i32(attn_lens_d_.as<int32_t>(), B, static_cast<int32_t>(fwd), st);
  launch_fill_i32(finished_d_.as<int32_t>(), B, 0, st);

  const bool use_graph = cfg_.use_cuda_graph != 0;
  if (use_graph) graph_.capture(st, {B, want_scores_}, [&] { launch_step(B); });

  // ---- GreedySearch::search host loop (decoding.cc:844-971) ----
  std::vector<std::vector<int32_t>> results(B);
  std::vector<double> score_sum(B, 0.0);
  std::vector<char> ended_by_eos(B, 0);
  std::vector<float> hscores;
  if (want_scores_) hscores.resize(static_cast<size_t>(total_steps) * B);
  std::vector<char> finished(B, 0);
  int64_t num_finished = 0;
  // The host looks at the sampled ids only where a row can finish: never without end tokens (the step count is known),
  // not before the first step at which some row is past min_length (DisableTokens masks the end ids until then,
  // decoding.cc:852-856), and from there every `poll` steps — the device marks finished rows itself (their K/V stream
  // stops), so a late look only costs a few steps of a shrinking batch.
  int64_t first_eos_step = total_steps;
  if (!r.end_ids.empty())
    for (int64_t b = 0; b < B; ++b)
      first_eos_step = std::min<int64_t>(first_eos_step, hstart[b] + std::max<int64_t>(0, r.min_length));
  const int64_t poll = eos_poll_interval();
  int32_t* hout = host_pinned_;     // reuse: [steps, B] sampled ids
  int64_t copied = 0;
  auto consume = [&](int64_t upto) {   // host bookkeeping for steps [copied, upto)
    CT2_CUDA_CHECK(cudaMemcpyAsync(hout + copied * B, out_d_.as<int32_t>() + copied * B,
                                   (upto - copied) * B * sizeof(int32_t), cudaMemcpyDeviceToHost, st));
    if (want_scores_)
      CT2_CUDA_CHECK(cudaMemcpyAsync(hscores.data() + copied * B, scores_d_.as<float>() + copied * B,
                                     (upto - copied) * B * sizeof(float), cudaMemcpyDeviceToHost, st));
    CT2_CUDA_CHECK(cudaStreamSynchronize(st));
    for (int64_t s = copied; s < upto; ++s) {
      for (int64_t b = 0; b < B; ++b) {
        if (finished[b]) continue;
        // step s consumed input token index fwd+s; its sample is a generated token only once the
        // prompt of row b is exhausted, i.e. fwd+s >= prompt_len-1
        if (fwd + s < r.prompt_lens[b] - 1) continue;
        const int32_t tok = hout[s * B + b];
        if (want_scores_) score_sum[b] += hscores[s * B + b];      // the end token's log-probability counts too
        const bool is_end = std::find(r.end_ids.begin(), r.end_ids.end(), tok) != r.end_ids.end();
        if (is_end) {
          if (r.return_end_token) results[b].push_back(tok);
          ended_by_eos[b] = 1;
          finished[b] = 1;
          ++num_finished;
        } else {
          results[b].push_back(tok);
          if (static_cast<int64_t>(results[b].size()) >= r.max_length) {
            finished[b] = 1;
            ++num_finished;
          }
        }
      }
    }
    copied = upto;
  };
  for (int64_t s = 0; s < total_steps && num_finished < B; ++s) {
    if (use_graph) {
      graph_.launch(st);
    } else {
      pdl_fence_next_launch();
      launch_step(B);
    }
    if (s + 1 == total_steps || (s >= first_eos_step && (s - first_eos_step) % poll == poll - 1)) consume(s + 1);
  }
  for (int64_t b = 0; b < B; ++b) {
    if (want_scores_) {
      // finalize_hypothesis_score (decoding.cc:189-203).  The reference decodes with include_eos_in_hypotheses = true
      // (decoding.h:154) and strips the end token afterwards (language_model.cc:253-257): the normalising length counts it.
      const double len = static_cast<double>(results[b].size()) + ((ended_by_eos[b] && !r.return_end_token) ? 1.0 : 0.0);
      out_scores[b] = static_cast<float>(len > 0 ? score_sum[b] / std::pow(len, static_cast<double>(r.length_penalty)) : score_sum[b]);
    }
    out_lens[b] = static_cast<int32_t>(results[b].size());
    for (int64_t t = 0; t < r.max_length; ++t)
      out_ids[b * r.max_length + t] = t < static_cast<int64_t>(results[b].size()) ? results[b][t] : -1;
  }
}

// Generator::generate_batch with beam_size > 1.  The decoder-only engine keeps contiguous per-row caches (its attention kernels
// stage whole 64-key boxes by TMA), so beams are reordered by re-gathering the rows into the second cache set after every step
// (Decoder::update_state does the same on every cached tensor); the search itself is the device-resident one of beam.h.
std::vector<TranslationHypotheses> Generator::generate_beam(const GenerationRequest& r) {
  std::lock_guard<std::mutex> lock(mu_);
  LlamaDecoder& d = *decoder_;
  cudaStream_t st = d.stream();
  const int64_t B = r.batch, P = r.max_prompt_len, L = r.max_length;
  const int beam = r.beam_size;
  const int64_t N = B * beam;
  CT2_REQUIRE(B > 0 && beam >= 2 && beam <= 32, "generate_beam: beam_size must be in [2, 32]");
  CT2_REQUIRE(N <= d.max_batch(), "generate_batch: batch x beam_size exceeds max_batch");
  CT2_REQUIRE(r.num_hypotheses >= 1 && r.num_hypotheses <= beam, "num_hypotheses must be in [1, beam_size]");
  CT2_REQUIRE(r.patience > 0.f && r.patience <= 2.f, "patience must be in (0, 2]");
  CT2_REQUIRE(L >= 1 && r.min_length <= L, "min_length is greater than max_length");
  CT2_REQUIRE(r.end_ids.size() <= 64, "at most 64 end tokens");
  for (int64_t b = 0; b < B; ++b)
    CT2_REQUIRE(r.prompt_lens[b] == P && P >= 1, "beam search needs prompts of equal length (at least the start token)");
  CT2_REQUIRE(P + L <= d.max_length(), "generate_batch: prompt + max_length exceeds max_length of the KV arena");
  if (!beam_) beam_ = std::make_unique<BeamSearchArena>();
  beam_->ensure(B, beam, L, dtype_size(d.dtype()));
  const int64_t V = d.config().vocab, fwd = P - 1;

  // prompt pass on B rows, then replicate_state: rows b -> b * beam + k
  int32_t* hp = host_pinned_;
  for (int64_t b = 0; b < B; ++b)
    for (int64_t t = 0; t < fwd; ++t) hp[b * fwd + t] = r.prompt_ids[b * P + t];
  int32_t* hend = hp + B * fwd;
  for (size_t i = 0; i < r.end_ids.size(); ++i) hend[i] = r.end_ids[i];
  if (fwd > 0) {
    CT2_CUDA_CHECK(cudaMemcpyAsync(prompt_d_.ptr, hp, B * fwd * sizeof(int32_t), cudaMemcpyHostToDevice, st));
    run_prefill(prompt_d_.as<int32_t>(), B, fwd);
    d.reorder_cache(nullptr, beam, N, fwd);
  }
  if (!r.end_ids.empty())
    CT2_CUDA_CHECK(cudaMemcpyAsync(beam_->end_ids.ptr, hend, r.end_ids.size() * 4, cudaMemcpyHostToDevice, st));
  BeamState bs = beam_->state(B, beam, V, L, r.min_length, r.patience, r.length_penalty, r.num_hypotheses,
                              static_cast<int>(r.end_ids.size()));
  // every row of entry b starts from its last prompt token
  std::vector<int32_t> start(N);
  for (int64_t n = 0; n < N; ++n) start[n] = r.prompt_ids[(n / beam) * P + P - 1];
  beam_->reset(bs, 0, d.dtype(), st);
  CT2_CUDA_CHECK(cudaMemcpyAsync(beam_->next_ids.ptr, start.data(), N * 4, cudaMemcpyHostToDevice, st));
  CT2_CUDA_CHECK(cudaStreamSynchronize(st));

  const int64_t poll = eos_poll_interval();
  const int64_t first_check = std::max<int64_t>(0, r.min_length);
  for (int64_t s = 0; s < L; ++s) {
    launch_fill_i32(lens_d_.as<int32_t>(), N, static_cast<int32_t>(fwd + s), st);
    d.forward_step(beam_->next_ids.as<int32_t>(), lens_d_.as<int32_t>(), N, d.logits_buffer());
    beam_->step(d.logits_buffer(), bs, d.dtype(), st);
    if (s + 1 == L) break;
    d.reorder_cache(beam_->parent.as<int32_t>(), beam, N, fwd + s + 1);
    if (s >= first_check && (s - first_check) % poll == poll - 1) {
      CT2_CUDA_CHECK(cudaMemcpyAsync(beam_->host, bs.num_finished, 4, cudaMemcpyDeviceToHost, st));
      CT2_CUDA_CHECK(cudaStreamSynchronize(st));
      if (*beam_->host >= B) break;
    }
  }
  auto out = beam_->collect(bs, r.length_penalty, r.num_hypotheses, r.return_end_token ? std::vector<int32_t>{} : r.end_ids, st);
  d.restore_cache_orientation();
  return out;
}

void Generator::forward(const int32_t* ids_h, int64_t batch, int64_t time, bool log_probs, float* logits_h) {
  std::lock_guard<std::mutex> lock(mu_);
  LlamaDecoder& d = *decoder_;
  cudaStream_t st = d.stream();
  CT2_REQUIRE(batch > 0 && batch <= d.max_batch() && time > 0 && time <= d.max_length(), "forward_batch: shape exceeds the arena");
  CT2_REQUIRE(batch * time <= d.prefill_chunk_rows(), "forward_batch: too many tokens for one pass");
  const int64_t V = d.config().vocab;
  CT2_CUDA_CHECK(cudaMemcpyAsync(prompt_d_.ptr, ids_h, batch * time * sizeof(int32_t), cudaMemcpyHostToDevice, st));
  CT2_CUDA_CHECK(cudaMemcpyAsync(ids_d_.ptr, prompt_d_.ptr, batch * time * sizeof(int32_t), cudaMemcpyDeviceToDevice, st));
  d.forward_prefill(ids_d_.as<int32_t>(), batch, time, 0, nullptr, nullptr, 0);
  // project max_batch rows at a time
  DeviceBuffer f32(static_cast<size_t>(d.max_batch()) * V * sizeof(float));
  DeviceBuffer rows_d(d.max_batch() * sizeof(int32_t));
  std::vector<int32_t> rows_h(d.max_batch());
  const int64_t total = batch * time;
  for (int64_t r0 = 0; r0 < total; r0 += d.max_batch()) {
    const int64_t n = std::min<int64_t>(d.max_batch(), total - r0);
    for (int64_t i = 0; i < n; ++i) rows_h[i] = static_cast<int32_t>(r0 + i);
    CT2_CUDA_CHECK(cudaMemcpyAsync(rows_d.ptr, rows_h.data(), n * sizeof(int32_t), cudaMemcpyHostToDevice, st));
    CT2_CUDA_CHECK(cudaStreamSynchronize(st));
    d.project_rows(rows_d.as<int32_t>(), n, d.logits_buffer());
    if (log_probs) launch_softmax(d.logits_buffer(), nullptr, n, V, true, d.logits_buffer(), d.dtype(), st);
    launch_convert_to_f32(d.logits_buffer(), n * V, f32.as<float>(), d.dtype(), st);
    CT2_CUDA_CHECK(cudaMemcpyAsync(logits_h + r0 * V, f32.ptr, n * V * sizeof(float), cudaMemcpyDeviceToHost, st));
    CT2_CUDA_CHECK(cudaStreamSynchronize(st));
  }
}

// Generator::score_batch (src/scoring.cc:6-66, language_model.cc:113-133): inputs = ids[:, :-1] go through the prompt pass
// in time chunks.  After each chunk, and before the next one overwrites the hidden state, the rows of its scored positions
// (offset <= t < len - 1: padding and positions before `offset` never reach the lm_head) are gathered into the slab; every
// full slab goes through the final RMSNorm + lm_head (project(): INT8 / AWQ / float heads, the prefill GEMM above 64 rows)
// and the fused LogSoftMax + Gather, which writes one float per position.  Only those floats come back to the host.
void Generator::score(const int32_t* ids_h, const int32_t* lens_h, int64_t batch, int64_t max_len, int64_t offset,
                      float* out_h) {
  std::lock_guard<std::mutex> lock(mu_);
  LlamaDecoder& d = *decoder_;
  cudaStream_t st = d.stream();
  CT2_REQUIRE(batch > 0 && batch <= d.max_batch(), "score_batch: batch size exceeds max_batch");
  CT2_REQUIRE(max_len >= 1 && max_len - 1 <= d.max_length(), "score_batch: sequences exceed max_length of the KV arena");
  CT2_REQUIRE(offset >= 0, "score_batch: offset must be >= 0");
  const int64_t T = max_len - 1;                       // input positions per row
  int64_t total = 0;
  for (int64_t b = 0; b < batch; ++b) {
    CT2_REQUIRE(lens_h[b] >= 0 && lens_h[b] <= max_len, "score_batch: a sequence length exceeds max_len");
    total += std::max<int64_t>(0, lens_h[b] - 1 - offset);
  }
  std::fill(out_h, out_h + batch * T, 0.f);
  if (total == 0) return;
  const int64_t V = d.config().vocab, dm = d.config().d_model, es = dtype_size(d.dtype());
  const int64_t cap = d.max_batch() * d.max_length();    // scored positions of the largest call
  if (!score_slab_.ptr) {
    // as many rows as 256 MB of logits hold, at least max_batch and at most one prompt-pass chunk
    score_slab_rows_ = std::min(d.prefill_chunk_rows(), std::max(d.max_batch(), (static_cast<int64_t>(256) << 20) / (V * es)));
    score_slab_.alloc(static_cast<size_t>(score_slab_rows_) * (V + dm) * es + 256);
    score_idx_d_.alloc(static_cast<size_t>(2) * cap * sizeof(int32_t));
    score_out_d_.alloc(static_cast<size_t>(cap) * sizeof(float));
    CT2_CUDA_CHECK(cudaMallocHost(&score_pinned_, static_cast<size_t>(2) * cap * sizeof(int32_t)));
  }
  uint8_t* logits = score_slab_.as<uint8_t>();
  uint8_t* hidden = logits + (static_cast<size_t>(score_slab_rows_) * V * es + 255) / 256 * 256;
  int32_t* rows_d = score_idx_d_.as<int32_t>();         // per scored position: its row in the chunk's hidden state
  int32_t* tgt_d = rows_d + cap;                        //                      and its target id
  int32_t* rows_h = score_pinned_;
  int32_t* tgt_h = score_pinned_ + cap;
  std::vector<int64_t> dest(total);                     // its place in out_h
  float* scores_d = score_out_d_.as<float>();

  CT2_CUDA_CHECK(cudaMemcpy2DAsync(prompt_d_.ptr, T * sizeof(int32_t), ids_h, max_len * sizeof(int32_t), T * sizeof(int32_t),
                                   batch, cudaMemcpyHostToDevice, st));
  int64_t picked = 0, done = 0;                         // positions gathered into the slab / projected and scored
  auto flush = [&](int64_t upto) {
    const int64_t n = upto - done;
    if (n == 0) return;
    d.project_hidden(hidden, n, logits);
    launch_log_softmax_gather(logits, tgt_d + done, n, V, scores_d + done, d.dtype(), st);
    done = upto;
  };
  run_prefill(prompt_d_.as<int32_t>(), batch, T, [&](int64_t t0, int64_t tc) {
    const int64_t first = picked;
    for (int64_t b = 0; b < batch; ++b)
      for (int64_t t = std::max(t0, offset); t < std::min<int64_t>(t0 + tc, lens_h[b] - 1); ++t) {
        rows_h[picked] = static_cast<int32_t>(b * tc + (t - t0));
        tgt_h[picked] = ids_h[b * max_len + t + 1];
        dest[picked++] = b * T + (t - offset);
      }
    if (picked == first) return;
    CT2_CUDA_CHECK(cudaMemcpyAsync(rows_d + first, rows_h + first, (picked - first) * sizeof(int32_t), cudaMemcpyHostToDevice, st));
    CT2_CUDA_CHECK(cudaMemcpyAsync(tgt_d + first, tgt_h + first, (picked - first) * sizeof(int32_t), cudaMemcpyHostToDevice, st));
    for (int64_t p = first; p < picked;) {
      const int64_t k = std::min(score_slab_rows_ - (p - done), picked - p);
      d.gather_hidden(rows_d + p, k, hidden + (p - done) * dm * es);
      p += k;
      if (p - done == score_slab_rows_) flush(p);
    }
  });
  flush(picked);
  std::vector<float> vals(total);
  CT2_CUDA_CHECK(cudaMemcpyAsync(vals.data(), scores_d, total * sizeof(float), cudaMemcpyDeviceToHost, st));
  CT2_CUDA_CHECK(cudaStreamSynchronize(st));
  for (int64_t i = 0; i < total; ++i) out_h[dest[i]] = vals[i];
}

void Generator::bench_decode(int64_t batch, int64_t prompt_len, int64_t steps, int64_t warmup, float* prefill_ms,
                             float* decode_ms, int64_t* launches) {
  std::lock_guard<std::mutex> lock(mu_);
  LlamaDecoder& d = *decoder_;
  cudaStream_t st = d.stream();
  CT2_REQUIRE(batch <= d.max_batch() && prompt_len + warmup + steps <= d.max_length(), "bench_decode: exceeds the arena");
  const int64_t V = d.config().vocab;
  // synthetic resident inputs: ids = (7919 * i) % V
  std::vector<int32_t> ids(batch * prompt_len);
  for (size_t i = 0; i < ids.size(); ++i) ids[i] = static_cast<int32_t>((7919ull * i + 3) % V);
  CT2_CUDA_CHECK(cudaMemcpy(prompt_d_.ptr, ids.data(), ids.size() * sizeof(int32_t), cudaMemcpyHostToDevice));
  int32_t gen[8] = {static_cast<int32_t>(prompt_len - 1), 0, 0, 0, INT32_MAX, 0, 0, 0};
  CT2_CUDA_CHECK(cudaMemcpy(step_d_.ptr, gen, sizeof(gen), cudaMemcpyHostToDevice));
  CT2_CUDA_CHECK(cudaDeviceSynchronize());      // pageable H2D: the DMA may still be running when cudaMemcpy returns (see upload())
  cudaEvent_t e0, e1, e2, e3;
  cudaEventCreate(&e0);
  cudaEventCreate(&e1);
  cudaEventCreate(&e2);
  cudaEventCreate(&e3);
  const int64_t fwd = prompt_len - 1;
  // warm-up prefill (first-use kernel configuration), then the timed one
  if (fwd > 0) run_prefill(prompt_d_.as<int32_t>(), batch, fwd);
  CT2_CUDA_CHECK(cudaStreamSynchronize(st));
  cudaEventRecord(e0, st);
  if (fwd > 0) run_prefill(prompt_d_.as<int32_t>(), batch, fwd);
  cudaEventRecord(e1, st);
  CT2_CUDA_CHECK(cudaMemcpy2DAsync(ids_d_.ptr, sizeof(int32_t), prompt_d_.as<int32_t>() + fwd, prompt_len * sizeof(int32_t),
                                   sizeof(int32_t), batch, cudaMemcpyDeviceToDevice, st));
  launch_fill_i32(lens_d_.as<int32_t>(), batch, static_cast<int32_t>(fwd), st);
  launch_fill_i32(attn_lens_d_.as<int32_t>(), batch, static_cast<int32_t>(fwd), st);
  launch_fill_i32(finished_d_.as<int32_t>(), batch, 0, st);
  const bool use_graph = cfg_.use_cuda_graph != 0;
  if (use_graph) graph_.capture(st, {batch, want_scores_}, [&] { launch_step(batch); });
  auto step = [&]() {
    if (use_graph)
      graph_.launch(st);
    else
      launch_step(batch);
  };
  for (int64_t s = 0; s < warmup; ++s) step();
  CT2_CUDA_CHECK(cudaStreamSynchronize(st));
  const int64_t l0 = g_kernel_launches.load();
  cudaProfilerStart();                 // ncu --profile-from-start off captures exactly the timed decode steps
  cudaEventRecord(e2, st);
  for (int64_t s = 0; s < steps; ++s) step();
  cudaEventRecord(e3, st);
  CT2_CUDA_CHECK(cudaStreamSynchronize(st));
  cudaProfilerStop();
  *launches = g_kernel_launches.load() - l0;
  cudaEventElapsedTime(prefill_ms, e0, e1);
  cudaEventElapsedTime(decode_ms, e2, e3);
  cudaEventDestroy(e0);
  cudaEventDestroy(e1);
  cudaEventDestroy(e2);
  cudaEventDestroy(e3);
}

void Generator::bench_last_logits(int64_t batch, float* logits_h, int64_t logits_len) {
  std::lock_guard<std::mutex> lock(mu_);
  LlamaDecoder& d = *decoder_;
  cudaStream_t st = d.stream();
  CT2_REQUIRE(batch >= 1 && batch <= d.max_batch(), "bench_last_logits: batch exceeds the arena");
  const int64_t V = d.config().vocab;
  CT2_REQUIRE(logits_len == batch * V, "bench_last_logits: the buffer must hold batch x vocab floats");
  DeviceBuffer f32(static_cast<size_t>(batch) * V * sizeof(float));
  launch_convert_to_f32(d.logits_buffer(), batch * V, f32.as<float>(), d.dtype(), st);
  CT2_CUDA_CHECK(cudaMemcpyAsync(logits_h, f32.ptr, batch * V * sizeof(float), cudaMemcpyDeviceToHost, st));
  CT2_CUDA_CHECK(cudaStreamSynchronize(st));
}

}  // namespace ct2b200
