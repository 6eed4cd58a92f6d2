# tools/ref_translate_attention.mk -- fixture tooling, not product code: builds tools/ref_translate_attention.cc against the
# CPU reference library that oracle/Makefile.ref builds, with that makefile's own defines, include paths and OpenMP runtime.
# The binary goes to a temporary directory; tools/make_golden.py runs it to write tests/golden/seq2seq_attention_ref.json
# and tests/test_oracle_translator_attention.py runs it live where the library has been built.
#
#   make -f tools/ref_translate_attention.mk [ATTN_OUT=/tmp/ct2ref_attention]

include oracle/Makefile.ref

ATTN_OUT ?= /tmp/ct2ref_attention

attention: $(ATTN_OUT)/ref_translate_attention

$(ATTN_OUT)/ref_translate_attention: tools/ref_translate_attention.cc $(OUT)/libct2ref.so
	@mkdir -p $(dir $@)
	$(CXX) -std=c++17 -O2 -w $(CT2_DEFS) $(CT2_INC) $< -o $@ $(GOMP) -L$(OUT) -lct2ref -Wl,-rpath,$(abspath $(OUT))

.PHONY: attention
