// ref_whisper_align.cc -- fixture generator, not product code: models::Whisper::align and ::detect_language of the unmodified
// reference (the CPU build of oracle/Makefile.ref, oracle/_ref/libct2ref.so; built by tools/ref_whisper_align.mk) for
// tools/make_golden.py (make_whisper_align_fixture).
//
//   stdin, line 1:  model_dir <TAB> compute_type
//   then one request per line, fields separated by tabs:
//     align <TAB> features.f32 <TAB> batch n_mels frames <TAB> median_filter_width <TAB> start ids <TAB> text rows <TAB> num_frames
//       (ids separated by single spaces, text rows separated by ';', one num_frames per entry)
//     lang <TAB> features.f32 <TAB> batch n_mels frames
//   stdout, per request: "ok" or "error <message>", then one line per entry:
//     align: "i,j i,j ..." <TAB> text_token_probs (%.9g)        lang: "token prob token prob ..." in the returned order
#include <cstdio>
#include <fstream>
#include <iostream>
#include <sstream>
#include <string>
#include <vector>

#include <ctranslate2/models/whisper.h>

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
    if (h.size() != 2) throw std::runtime_error("header: model_dir, compute_type");
    ctranslate2::models::ModelLoader loader(h[0]);
    loader.device = ctranslate2::Device::CPU;
    loader.compute_type = ctranslate2::str_to_compute_type(h[1]);
    ctranslate2::ReplicaPoolConfig config;
    config.num_threads_per_replica = 2;
    ctranslate2::models::Whisper whisper(loader, config);
    for (std::string line; std::getline(std::cin, line);) {
      const std::vector<std::string> f = split(line, '\t');
      try {
        if (f.at(0) == "align") {
          std::vector<std::vector<size_t>> text;
          for (const auto& row : split(f.at(5), ';')) text.push_back(ids(row));
          if (f.at(5).empty()) text.clear();
          auto futures = whisper.align(features(f.at(1), f.at(2)), ids(f.at(4)), text, ids(f.at(6)), std::stol(f.at(3)));
          std::vector<ctranslate2::models::WhisperAlignmentResult> res;
          for (auto& fu : futures) res.push_back(fu.get());
          std::printf("ok\n");
          for (const auto& r : res) {
            for (size_t i = 0; i < r.alignments.size(); ++i)
              std::printf("%s%lld,%lld", i ? " " : "", static_cast<long long>(r.alignments[i].first),
                          static_cast<long long>(r.alignments[i].second));
            std::printf("\t");
            for (size_t i = 0; i < r.text_token_probs.size(); ++i) std::printf("%s%.9g", i ? " " : "", r.text_token_probs[i]);
            std::printf("\n");
          }
        } else if (f.at(0) == "lang") {
          auto futures = whisper.detect_language(features(f.at(1), f.at(2)));
          std::vector<std::vector<std::pair<std::string, float>>> res;
          for (auto& fu : futures) res.push_back(fu.get());
          std::printf("ok\n");
          for (const auto& r : res) {
            for (size_t i = 0; i < r.size(); ++i) std::printf("%s%s %.9g", i ? " " : "", r[i].first.c_str(), r[i].second);
            std::printf("\n");
          }
        } else {
          throw std::runtime_error("unknown request " + f.at(0));
        }
      } catch (const std::exception& e) {
        std::printf("error %s\n", e.what());
      }
      std::fflush(stdout);
    }
  } catch (const std::exception& e) {
    std::fprintf(stderr, "ref_whisper_align: %s\n", e.what());
    return 1;
  }
  return 0;
}
