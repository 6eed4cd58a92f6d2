// ref_encoder.cc -- fixture generator, not product code: ctranslate2::Encoder::forward_batch of the unmodified reference (the
// CPU build of oracle/Makefile.ref, oracle/_ref/libct2ref.so; built by tools/ref_encoder.mk) on ids, for
// tools/make_golden.py (make_encoder_fixture).
//
//   stdin, line 1:  model_dir <TAB> compute_type
//   then one row per line:  ids <TAB> token type ids  (separated by single spaces; types empty on every line = none given)
//   stdout: one line per row, in order:  last_hidden_state of the row's valid positions <TAB> pooler_output (%.9g, flattened;
//   the second field is empty without a pooler)
#include <cstdio>
#include <iostream>
#include <sstream>
#include <string>
#include <vector>

#include <ctranslate2/encoder.h>

namespace {

std::vector<size_t> parse_ids(const std::string& s) {
  std::vector<size_t> out;
  std::istringstream in(s);
  for (size_t v; in >> v;) out.push_back(v);
  return out;
}

}  // namespace

int main() {
  try {
    std::string header;
    std::getline(std::cin, header);
    const size_t tab = header.find('\t');
    if (tab == std::string::npos) throw std::runtime_error("header: model_dir, compute_type");
    std::vector<std::vector<size_t>> ids, types;
    bool any_types = false;
    for (std::string line; std::getline(std::cin, line);) {
      const size_t t = line.find('\t');
      if (t == std::string::npos) throw std::runtime_error("row lines need a tab");
      ids.push_back(parse_ids(line.substr(0, t)));
      types.push_back(parse_ids(line.substr(t + 1)));
      any_types = any_types || !types.back().empty();
    }
    if (!any_types) types.clear();
    ctranslate2::models::ModelLoader loader(header.substr(0, tab));
    loader.device = ctranslate2::Device::CPU;
    loader.compute_type = ctranslate2::str_to_compute_type(header.substr(tab + 1));
    ctranslate2::ReplicaPoolConfig config;
    config.num_threads_per_replica = 2;
    ctranslate2::Encoder encoder(loader, config);
    const ctranslate2::EncoderForwardOutput out = encoder.forward_batch_async(ids, types).get();
    const ctranslate2::StorageView hidden = out.last_hidden_state.to_float32();
    const std::vector<float> h = hidden.to_vector<float>();
    const size_t T = hidden.dim(1), d = hidden.dim(2);
    std::vector<float> p;
    if (out.pooler_output) p = out.pooler_output->to_float32().to_vector<float>();
    for (size_t b = 0; b < ids.size(); ++b) {
      for (size_t i = 0; i < ids[b].size() * d; ++i) std::printf("%s%.9g", i ? " " : "", h[b * T * d + i]);
      std::printf("\t");
      for (size_t i = 0; i < (p.empty() ? 0 : d); ++i) std::printf("%s%.9g", i ? " " : "", p[b * d + i]);
      std::printf("\n");
    }
  } catch (const std::exception& e) {
    std::fprintf(stderr, "ref_encoder: %s\n", e.what());
    return 1;
  }
  return 0;
}
