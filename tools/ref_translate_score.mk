# tools/ref_translate_score.mk -- fixture tooling, not product code: builds tools/ref_translate_score.cc against the CPU
# reference library that oracle/Makefile.ref builds, with that makefile's own defines, include paths and OpenMP runtime.
# The binary goes to a temporary directory; tools/make_golden.py runs it to write tests/golden/seq2seq_score_ref.json.
#
#   make -f tools/ref_translate_score.mk [SCORE_OUT=/tmp/ct2ref_score]

include oracle/Makefile.ref

SCORE_OUT ?= /tmp/ct2ref_score

score: $(SCORE_OUT)/ref_translate_score

$(SCORE_OUT)/ref_translate_score: tools/ref_translate_score.cc $(OUT)/libct2ref.so
	@mkdir -p $(dir $@)
	$(CXX) -std=c++17 -O2 -w $(CT2_DEFS) $(CT2_INC) $< -o $@ $(GOMP) -L$(OUT) -lct2ref -Wl,-rpath,$(abspath $(OUT))

.PHONY: score
