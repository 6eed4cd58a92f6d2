// ref_translate_score.cc -- fixture generator, not product code: ctranslate2::Translator::score_batch of the unmodified
// reference (the CPU build of oracle/Makefile.ref, oracle/_ref/libct2ref.so; built by tools/ref_translate_score.mk) on token
// strings, for tools/make_golden.py (make_translator_score_fixture).
//
//   stdin, line 1:  model_dir <TAB> compute_type <TAB> max_input_length <TAB> offset <TAB> max_batch_size
//   then one pair per line:  source tokens <TAB> target tokens  (tokens separated by single spaces; either side may be empty)
//   stdout: one line per pair, in order:  scored tokens <TAB> log-probabilities (%.9g)
#include <cstdio>
#include <iostream>
#include <sstream>
#include <string>
#include <vector>

#include <ctranslate2/translator.h>

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

}  // namespace

int main() {
  try {
    std::string header;
    std::getline(std::cin, header);
    const std::vector<std::string> h = split(header, '\t');
    if (h.size() != 5) throw std::runtime_error("header: model_dir, compute_type, max_input_length, offset, max_batch_size");
    std::vector<std::vector<std::string>> source, target;
    for (std::string line; std::getline(std::cin, line);) {
      const size_t tab = line.find('\t');
      if (tab == std::string::npos) throw std::runtime_error("pair lines need a tab");
      source.push_back(split(line.substr(0, tab), ' '));
      target.push_back(split(line.substr(tab + 1), ' '));
    }
    ctranslate2::models::ModelLoader loader(h[0]);
    loader.device = ctranslate2::Device::CPU;
    loader.compute_type = ctranslate2::str_to_compute_type(h[1]);
    ctranslate2::ReplicaPoolConfig config;
    config.num_threads_per_replica = 2;
    ctranslate2::Translator translator(loader, config);
    ctranslate2::ScoringOptions options;
    options.max_input_length = std::stoul(h[2]);
    options.offset = std::stol(h[3]);
    const auto results = translator.score_batch(source, target, options, std::stoul(h[4]));
    for (const auto& r : results) {
      for (size_t i = 0; i < r.tokens.size(); ++i) std::printf("%s%s", i ? " " : "", r.tokens[i].c_str());
      std::printf("\t");
      for (size_t i = 0; i < r.tokens_score.size(); ++i) std::printf("%s%.9g", i ? " " : "", r.tokens_score[i]);
      std::printf("\n");
    }
  } catch (const std::exception& e) {
    std::fprintf(stderr, "ref_translate_score: %s\n", e.what());
    return 1;
  }
  return 0;
}
