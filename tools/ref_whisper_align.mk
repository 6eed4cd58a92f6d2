# tools/ref_whisper_align.mk -- fixture tooling, not product code: builds tools/ref_whisper_align.cc against the CPU reference
# library that oracle/Makefile.ref builds, with that makefile's own defines, include paths and OpenMP runtime.  The binary goes
# to a temporary directory; tools/make_golden.py runs it to write tests/golden/whisper_align_ref.json.
#
#   make -f tools/ref_whisper_align.mk [ALIGN_OUT=/tmp/ct2ref_align]

include oracle/Makefile.ref

ALIGN_OUT ?= /tmp/ct2ref_align

align: $(ALIGN_OUT)/ref_whisper_align

$(ALIGN_OUT)/ref_whisper_align: tools/ref_whisper_align.cc $(OUT)/libct2ref.so
	@mkdir -p $(dir $@)
	$(CXX) -std=c++17 -O2 -w $(CT2_DEFS) $(CT2_INC) $< -o $@ $(GOMP) -L$(OUT) -lct2ref -Wl,-rpath,$(abspath $(OUT))

.PHONY: align
