# oracle/lazy_blend.mk — builds the checker of the windowed blend (test infrastructure, never the product):
#
#   make -f lazy_blend.mk ref -> oracle/_ref/lazy_blend_test   pano_host.hh's B200LazyBlender next to the reference's
#                                                              LinearBlender / MultiBandBlender (tests/test_gpu_blend_stream.py)
# Needs oracle/Makefile's `ref` (libopenpano_ref.so, which holds the reference's blender TUs) and
# openpano_b200/libpano_b200.so first.  Flags are oracle/Makefile's parity flags; outputs go to oracle/_ref/ only.

REF ?= /root/reference
SRC := $(REF)/src
HERE := $(dir $(abspath $(lastword $(MAKEFILE_LIST))))
OUT := $(HERE)_ref
PANO_DIR := $(HERE)../openpano_b200
REF_INC := -I $(SRC) -I $(SRC)/lib -isystem $(SRC)/third-party -I $(HERE)refshim/eigen_stub

.PHONY: ref
ref:
	@if [ -d "$(SRC)" ]; then $(MAKE) -f $(HERE)lazy_blend.mk $(OUT)/lazy_blend_test; \
	 else echo "oracle/lazy_blend.mk: $(SRC) not present, keeping the prebuilt oracle/_ref/lazy_blend_test"; fi

$(OUT)/lazy_blend_test: $(HERE)../tests/adaptor/lazy_blend_test.cc $(PANO_DIR)/host/pano_host.hh $(HERE)../include/pano_b200.h $(OUT)/libopenpano_ref.so
	g++ -std=c++11 -O1 -ffp-contract=off -msse3 -w -DDISABLE_JPEG $(REF_INC) -I $(HERE)../include -I $(PANO_DIR)/host \
	  -o $@ $< -L $(OUT) -lopenpano_ref -L $(PANO_DIR) -lpano_b200 \
	  -Wl,-rpath,'$$ORIGIN' -Wl,-rpath,'$$ORIGIN/../../openpano_b200'
