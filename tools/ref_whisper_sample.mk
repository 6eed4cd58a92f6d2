# tools/ref_whisper_sample.mk -- fixture tooling, not product code: builds tools/ref_whisper_sample.cc against the CPU reference
# library that oracle/Makefile.ref builds, with that makefile's own defines, include paths and OpenMP runtime.  The binary goes
# to a temporary directory; tools/make_golden.py runs it to write tests/golden/whisper_sampling_ref.json.
#
#   make -f tools/ref_whisper_sample.mk [SAMPLE_OUT=/tmp/ct2ref_sample]

include oracle/Makefile.ref

SAMPLE_OUT ?= /tmp/ct2ref_sample

sample: $(SAMPLE_OUT)/ref_whisper_sample

$(SAMPLE_OUT)/ref_whisper_sample: tools/ref_whisper_sample.cc $(OUT)/libct2ref.so
	@mkdir -p $(dir $@)
	$(CXX) -std=c++17 -O2 -w $(CT2_DEFS) $(CT2_INC) $< -o $@ $(GOMP) -L$(OUT) -lct2ref -Wl,-rpath,$(abspath $(OUT))

.PHONY: sample
