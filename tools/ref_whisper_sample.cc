// ref_whisper_sample.cc -- fixture generator, not product code: models::Whisper::generate with random sampling of the
// unmodified reference (the CPU build of oracle/Makefile.ref, oracle/_ref/libct2ref.so; built by tools/ref_whisper_sample.mk)
// for tools/make_golden.py (make_whisper_sampling_fixture).
//
//   stdin, line 1:  model_dir <TAB> compute_type <TAB> seed   (ctranslate2::set_random_seed before the model is loaded)
//   then one request per line, fields separated by tabs:
//     features.f32 <TAB> batch n_mels frames <TAB> prompt rows <TAB> sampling_topk <TAB> sampling_temperature <TAB>
//     num_hypotheses <TAB> length_penalty <TAB> max_length
//       (ids separated by single spaces, prompt rows separated by ';'; beam_size 1, return_scores)
//   stdout, per request: "ok" or "error <message>", then one line per hypothesis of every entry:
//     entry <TAB> score (%.9g) <TAB> ids separated by spaces
#include <cstdio>
#include <fstream>
#include <iostream>
#include <sstream>
#include <string>
#include <vector>

#include <ctranslate2/models/whisper.h>
#include <ctranslate2/random.h>

namespace {

std::vector<std::string> split(const std::string& s, char sep) {
  std::vector<std::string> out;
  if (s.empty()) return out;
  std::string cur;
  std::istringstream in(s);
  while (std::getline(in, cur, sep)) out.push_back(cur);
  if (s.back() == sep) out.emplace_back();
  return out;
}

std::vector<size_t> ids(const std::string& s) {
  std::vector<size_t> out;
  for (const auto& t : split(s, ' '))
    if (!t.empty()) out.push_back(std::stoul(t));
  return out;
}

ctranslate2::StorageView features(const std::string& path, const std::string& dims) {
  const std::vector<size_t> d = ids(dims);
  if (d.size() != 3) throw std::runtime_error("features need 3 dimensions");
  std::vector<float> v(d[0] * d[1] * d[2]);
  std::ifstream f(path, std::ios::binary);
  f.read(reinterpret_cast<char*>(v.data()), v.size() * sizeof(float));
  if (!f) throw std::runtime_error("cannot read " + path);
  return ctranslate2::StorageView({static_cast<ctranslate2::dim_t>(d[0]), static_cast<ctranslate2::dim_t>(d[1]),
                                   static_cast<ctranslate2::dim_t>(d[2])}, v);
}

}  // namespace

int main() {
  try {
    std::string header;
    std::getline(std::cin, header);
    const std::vector<std::string> h = split(header, '\t');
    if (h.size() != 3) throw std::runtime_error("header: model_dir, compute_type, seed");
    ctranslate2::set_random_seed(static_cast<unsigned int>(std::stoul(h[2])));
    ctranslate2::models::ModelLoader loader(h[0]);
    loader.device = ctranslate2::Device::CPU;
    loader.compute_type = ctranslate2::str_to_compute_type(h[1]);
    ctranslate2::ReplicaPoolConfig config;
    config.num_threads_per_replica = 1;
    ctranslate2::models::Whisper whisper(loader, config);
    for (std::string line; std::getline(std::cin, line);) {
      const std::vector<std::string> f = split(line, '\t');
      try {
        std::vector<std::vector<size_t>> prompts;
        for (const auto& row : split(f.at(2), ';')) prompts.push_back(ids(row));
        ctranslate2::models::WhisperOptions o;
        o.beam_size = 1;
        o.sampling_topk = std::stoul(f.at(3));
        o.sampling_temperature = std::stof(f.at(4));
        o.num_hypotheses = std::stoul(f.at(5));
        o.length_penalty = std::stof(f.at(6));
        o.max_length = std::stoul(f.at(7));
        o.return_scores = true;
        auto futures = whisper.generate(features(f.at(0), f.at(1)), prompts, o);
        std::vector<ctranslate2::models::WhisperGenerationResult> res;
        for (auto& fu : futures) res.push_back(fu.get());
        std::printf("ok\n");
        for (size_t b = 0; b < res.size(); ++b)
          for (size_t j = 0; j < res[b].sequences_ids.size(); ++j) {
            std::printf("%zu\t%.9g\t", b, res[b].scores[j]);
            const auto& s = res[b].sequences_ids[j];
            for (size_t i = 0; i < s.size(); ++i) std::printf("%s%zu", i ? " " : "", s[i]);
            std::printf("\n");
          }
      } catch (const std::exception& e) {
        std::printf("error %s\n", e.what());
      }
      std::fflush(stdout);
    }
  } catch (const std::exception& e) {
    std::fprintf(stderr, "ref_whisper_sample: %s\n", e.what());
    return 1;
  }
  return 0;
}
