// ref_translate_attention.cc -- fixture generator, not product code: ctranslate2::Translator::translate_batch of the
// unmodified reference (the CPU build of oracle/Makefile.ref, oracle/_ref/libct2ref.so; built by
// tools/ref_translate_attention.mk) with return_attention, replace_unknowns and coverage_penalty, on token strings, for
// tools/make_golden.py (make_seq2seq_attention_fixture).
//
//   stdin, line 1:  model_dir <TAB> compute_type
//   then one request per line, tab-separated:
//     beam_size, num_hypotheses, length_penalty, max_decoding_length, min_decoding_length, coverage_penalty,
//     return_end_token, return_attention, replace_unknowns (each 0 / 1), sources
//   where sources is a list separated by '|' of token lists separated by single spaces.
//   stdout, per request: one line per source, in order:
//     hypotheses ('|'-separated token lists) <TAB> scores (%.9g) <TAB> attention
//   where the attention holds one matrix per hypothesis separated by '|', rows separated by ';', values (%.9g) by spaces.
//   A request the reference refuses prints one line "ERROR <TAB> message" instead.
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

std::vector<std::vector<std::string>> split_lists(const std::string& s) {
  std::vector<std::vector<std::string>> out;
  for (const auto& part : split(s, '|')) out.push_back(split(part, ' '));
  return out;
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
    ctranslate2::Translator translator(loader, config);
    for (std::string line; std::getline(std::cin, line);) {
      const std::vector<std::string> f = split(line, '\t');
      if (f.size() != 10) throw std::runtime_error("request lines have 10 fields");
      ctranslate2::TranslationOptions options;
      options.beam_size = std::stoul(f[0]);
      options.num_hypotheses = std::stoul(f[1]);
      options.length_penalty = std::stof(f[2]);
      options.max_decoding_length = std::stoul(f[3]);
      options.min_decoding_length = std::stoul(f[4]);
      options.coverage_penalty = std::stof(f[5]);
      options.return_end_token = f[6] == "1";
      options.return_attention = f[7] == "1";
      options.replace_unknowns = f[8] == "1";
      options.return_scores = true;
      const auto source = split_lists(f[9]);
      std::vector<ctranslate2::TranslationResult> results;
      try {
        results = translator.translate_batch(source, options);
      } catch (const std::exception& e) {
        std::printf("ERROR\t%s\n", e.what());
        continue;
      }
      for (const auto& r : results) {
        for (size_t k = 0; k < r.hypotheses.size(); ++k) {
          std::printf("%s", k ? "|" : "");
          for (size_t i = 0; i < r.hypotheses[k].size(); ++i) std::printf("%s%s", i ? " " : "", r.hypotheses[k][i].c_str());
        }
        std::printf("\t");
        for (size_t k = 0; k < r.scores.size(); ++k) std::printf("%s%.9g", k ? " " : "", r.scores[k]);
        std::printf("\t");
        for (size_t k = 0; k < r.attention.size(); ++k) {
          std::printf("%s", k ? "|" : "");
          for (size_t t = 0; t < r.attention[k].size(); ++t) {
            std::printf("%s", t ? ";" : "");
            for (size_t s = 0; s < r.attention[k][t].size(); ++s) std::printf("%s%.9g", s ? " " : "", r.attention[k][t][s]);
          }
        }
        std::printf("\n");
      }
    }
  } catch (const std::exception& e) {
    std::fprintf(stderr, "ref_translate_attention: %s\n", e.what());
    return 1;
  }
  return 0;
}
