# oracle/cyl_blend.mk — builds the checker of cylinder mode's blend from unwarped images (test infrastructure,
# never the product):
#
#   make -f cyl_blend.mk ref -> oracle/_ref/cyl_blend_test   pano_host.hh's B200CylinderBlender next to the reference's
#                                                            CylinderWarper + LinearBlender / MultiBandBlender
#                                                            (tests/test_gpu_blend_cyl.py)
# Needs oracle/Makefile's `ref` (libopenpano_ref.so, which holds the reference's warper and blender TUs) and
# openpano_b200/libpano_b200.so first.  Flags are oracle/Makefile's parity flags; outputs go to oracle/_ref/ only.

REF ?= /root/reference
SRC := $(REF)/src
HERE := $(dir $(abspath $(lastword $(MAKEFILE_LIST))))
OUT := $(HERE)_ref
PANO_DIR := $(HERE)../openpano_b200
REF_INC := -I $(SRC) -I $(SRC)/lib -isystem $(SRC)/third-party -I $(HERE)refshim/eigen_stub

.PHONY: ref
ref:
	@if [ -d "$(SRC)" ]; then $(MAKE) -f $(HERE)cyl_blend.mk $(OUT)/cyl_blend_test; \
	 else echo "oracle/cyl_blend.mk: $(SRC) not present, keeping the prebuilt oracle/_ref/cyl_blend_test"; fi

$(OUT)/cyl_blend_test: $(HERE)../tests/adaptor/cyl_blend_test.cc $(PANO_DIR)/host/pano_host.hh $(HERE)../include/pano_b200.h $(OUT)/libopenpano_ref.so
	g++ -std=c++11 -O1 -ffp-contract=off -msse3 -w -DDISABLE_JPEG $(REF_INC) -I $(HERE)../include -I $(PANO_DIR)/host \
	  -o $@ $< -L $(OUT) -lopenpano_ref -L $(PANO_DIR) -lpano_b200 \
	  -Wl,-rpath,'$$ORIGIN' -Wl,-rpath,'$$ORIGIN/../../openpano_b200'
