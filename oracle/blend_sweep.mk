# oracle/blend_sweep.mk — builds the checker of the blend-sweep mosaic writer (test infrastructure, never the
# product):
#
#   make -f blend_sweep.mk ref -> oracle/_ref/blend_sweep_test    pano_host_io.hh's B200PixelBlender::write_sweep
#                                                                  next to the reference's blenders, crop and
#                                                                  write_rgb (tests/test_gpu_blend_sweep.py)
# Needs oracle/Makefile's `ref` (libopenpano_ref.so, which holds the reference's blenders, imgio.cc and lodepng)
# and openpano_b200/libpano_b200.so first.  Flags are oracle/Makefile's parity flags; outputs go to oracle/_ref/ only.

REF ?= /root/reference
SRC := $(REF)/src
HERE := $(dir $(abspath $(lastword $(MAKEFILE_LIST))))
OUT := $(HERE)_ref
PANO_DIR := $(HERE)../openpano_b200
REF_INC := -I $(SRC) -I $(SRC)/lib -isystem $(SRC)/third-party -I $(HERE)refshim/eigen_stub

.PHONY: ref
ref:
	@if [ -d "$(SRC)" ]; then $(MAKE) -f $(HERE)blend_sweep.mk $(OUT)/blend_sweep_test; \
	 else echo "oracle/blend_sweep.mk: $(SRC) not present, keeping the prebuilt oracle/_ref/blend_sweep_test"; fi

$(OUT)/blend_sweep_test: $(HERE)../tests/adaptor/blend_sweep_test.cc $(PANO_DIR)/host/pano_host.hh $(PANO_DIR)/host/pano_host_io.hh $(HERE)../include/pano_b200.h $(OUT)/libopenpano_ref.so
	g++ -std=c++11 -O1 -ffp-contract=off -msse3 -w -DDISABLE_JPEG $(REF_INC) -I $(HERE)../include \
	  -I $(PANO_DIR)/host -o $@ $< -L $(OUT) -lopenpano_ref -L $(PANO_DIR) -lpano_b200 -lpthread \
	  -Wl,-rpath,'$$ORIGIN' -Wl,-rpath,'$$ORIGIN/../../openpano_b200'
