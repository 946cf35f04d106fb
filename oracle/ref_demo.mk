# Test-infrastructure only, beside Makefile (run after it: `make -C oracle -f ref_demo.mk`).
#
#   _ref/ref_demo   the reference's demo program (test/test.cpp: Harvest, CheapTrick, D4C, ParameterModification --
#                   f0 scaling and spectral stretch from argv[3] / argv[4] -- then three syntheses), compiled
#                   UNCHANGED from where it lies with src/synthesisrealtime.cpp beside it, against
#                   _ref/libworld_ref.so (which holds tools/audioio.cpp), with the reference's flags.
#                   tests/test_*_modify.py run it on the fixture and compare its output with the library's chain.
#                   Only built when the reference tree is present; the GPU box uses the prebuilt file.
#
# Nothing under world_b200/ (the product) links, loads or calls it.
REF ?= /root/reference
CXX ?= g++
REF_FLAGS = -O1 -fPIC -w

demo:
	@if [ -d $(REF)/test ] && [ -f _ref/libworld_ref.so ]; then $(MAKE) -f ref_demo.mk _ref/ref_demo; \
	 else echo "oracle: reference demo or _ref/libworld_ref.so absent - keeping prebuilt _ref/ref_demo (if any)"; fi

_ref/ref_demo: $(REF)/test/test.cpp $(REF)/src/synthesisrealtime.cpp _ref/libworld_ref.so ref_demo.mk
	$(CXX) $(REF_FLAGS) -I$(REF)/src -I$(REF)/tools -o $@ $(REF)/test/test.cpp $(REF)/src/synthesisrealtime.cpp \
	  -L_ref -lworld_ref -Wl,-rpath,'$$ORIGIN' -lm

.PHONY: demo
