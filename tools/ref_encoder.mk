# tools/ref_encoder.mk -- fixture tooling, not product code: builds tools/ref_encoder.cc against the CPU reference library
# that oracle/Makefile.ref builds, with that makefile's own defines, include paths and OpenMP runtime.  The binary goes to a
# temporary directory; tools/make_golden.py --encoder-only runs it to write tests/golden/encoder_ref.json.
#
#   make -f tools/ref_encoder.mk [ENCODER_OUT=/tmp/ct2ref_encoder]

include oracle/Makefile.ref

ENCODER_OUT ?= /tmp/ct2ref_encoder

encoder: $(ENCODER_OUT)/ref_encoder

$(ENCODER_OUT)/ref_encoder: tools/ref_encoder.cc $(OUT)/libct2ref.so
	@mkdir -p $(dir $@)
	$(CXX) -std=c++17 -O2 -w $(CT2_DEFS) $(CT2_INC) $< -o $@ $(GOMP) -L$(OUT) -lct2ref -Wl,-rpath,$(abspath $(OUT))

.PHONY: encoder
