# oracle/lazy_sift.mk — builds the checker of the windowed SIFT (test infrastructure, never the product):
#
#   make -f lazy_sift.mk ref -> oracle/_ref/lazy_sift_test   pano_host.hh's B200SIFTDetector::detect_lazy next to the
#                                                            reference's calc_feature loop (ImageRef::load + SIFTDetector::
#                                                            detect_feature) on PPM / PGM files (tests/test_gpu_sift_stream.py)
# Needs oracle/Makefile's `ref` (libopenpano_ref.so, which holds the reference's imgio and SIFT TUs) and
# openpano_b200/libpano_b200.so first.  Flags are oracle/Makefile's parity flags; outputs go to oracle/_ref/ only.

REF ?= /root/reference
SRC := $(REF)/src
HERE := $(dir $(abspath $(lastword $(MAKEFILE_LIST))))
OUT := $(HERE)_ref
PANO_DIR := $(HERE)../openpano_b200
REF_INC := -I $(SRC) -I $(SRC)/lib -isystem $(SRC)/third-party -I $(HERE)refshim/eigen_stub

.PHONY: ref
ref:
	@if [ -d "$(SRC)" ]; then $(MAKE) -f $(HERE)lazy_sift.mk $(OUT)/lazy_sift_test; \
	 else echo "oracle/lazy_sift.mk: $(SRC) not present, keeping the prebuilt oracle/_ref/lazy_sift_test"; fi

$(OUT)/lazy_sift_test: $(HERE)../tests/adaptor/lazy_sift_test.cc $(PANO_DIR)/host/pano_host.hh $(HERE)../include/pano_b200.h $(OUT)/libopenpano_ref.so
	g++ -std=c++11 -O1 -ffp-contract=off -msse3 -w -DDISABLE_JPEG $(REF_INC) -I $(HERE)../include -I $(PANO_DIR)/host \
	  -o $@ $< -L $(OUT) -lopenpano_ref -L $(PANO_DIR) -lpano_b200 \
	  -Wl,-rpath,'$$ORIGIN' -Wl,-rpath,'$$ORIGIN/../../openpano_b200'
