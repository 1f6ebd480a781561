# oracle/cyl_sweep.mk — builds the checkers of cylinder mode's perspective correction,
# CylinderStitcher::perspective_correction (stitch/cylstitcher.cc:139-180) (test infrastructure, never the product),
# next to what oracle/Makefile builds:
#
#   make -f cyl_sweep.mk oracle -> oracle/liboracle_persp.so              plain-C restatement (orc_persp.c)
#   make -f cyl_sweep.mk ref    -> oracle/_ref/libopenpano_ref_persp.so   the reference's own perspective_correction
#                                                                         (refshim/ref_persp.cc)
#                                  oracle/_ref/cyl_sweep_test             pano_host_io.hh's
#                                                                         B200CylinderBlender::write_sweep next to
#                                                                         the reference (tests/test_gpu_cyl_sweep.py)
# `ref` needs oracle/Makefile's `ref` (libopenpano_ref.so) and openpano_b200/libpano_b200.so first.  Flags are
# oracle/Makefile's parity flags; the reference sources are compiled IN PLACE, outputs go to oracle/_ref/ only.  With hidden visibility, one section
# per function and --gc-sections the linker keeps perspective_correction and what it calls; --no-undefined makes a
# symbol that is still missing a build error instead of a load-time one.

REF ?= /root/reference
SRC := $(REF)/src
HERE := $(dir $(abspath $(lastword $(MAKEFILE_LIST))))
OUT := $(HERE)_ref
REF_INC := -I $(SRC) -I $(SRC)/lib -isystem $(SRC)/third-party -I $(HERE)refshim/eigen_stub
CC ?= gcc

.PHONY: all oracle ref
all: oracle ref

oracle: $(HERE)liboracle_persp.so
$(HERE)liboracle_persp.so: $(HERE)orc_persp.c $(HERE)persp_api.h $(HERE)orc_common.h
	$(CC) -std=gnu11 -O2 -ffp-contract=off -msse3 -fPIC -shared -Wall -Wno-unused-function -o $@ $(HERE)orc_persp.c -lm

ref:
	@if [ -d "$(SRC)" ]; then $(MAKE) -f $(HERE)cyl_sweep.mk $(OUT)/libopenpano_ref_persp.so $(OUT)/cyl_sweep_test; \
	 else echo "oracle/cyl_sweep.mk: $(SRC) not present, keeping prebuilt oracle/_ref cylinder-sweep checkers"; fi

$(OUT)/libopenpano_ref_persp.so: $(HERE)refshim/ref_persp.cc $(HERE)persp_api.h $(OUT)/libopenpano_ref.so
	g++ -std=c++11 -fPIC -shared -w -DDISABLE_JPEG $(REF_INC) -O2 -ffp-contract=off -msse3 \
	  -fvisibility=hidden -ffunction-sections -fdata-sections -o $@ $(HERE)refshim/ref_persp.cc \
	  -Wl,--gc-sections -Wl,--no-undefined -L $(OUT) -lopenpano_ref -Wl,-rpath,'$$ORIGIN'

# pano_host_io.hh's B200CylinderBlender::write_sweep next to the reference's warp, blenders,
# perspective_correction, crop and write_rgb (tests/test_gpu_cyl_sweep.py).  Needs openpano_b200/libpano_b200.so.
PANO_DIR := $(HERE)../openpano_b200
$(OUT)/cyl_sweep_test: $(HERE)../tests/adaptor/cyl_sweep_test.cc $(PANO_DIR)/host/pano_host.hh $(PANO_DIR)/host/pano_host_io.hh $(HERE)../include/pano_b200.h $(HERE)persp_api.h $(OUT)/libopenpano_ref_persp.so
	g++ -std=c++11 -O1 -ffp-contract=off -msse3 -w -DDISABLE_JPEG $(REF_INC) -I $(HERE)../include -I $(HERE) \
	  -I $(PANO_DIR)/host -o $@ $< -L $(OUT) -lopenpano_ref_persp -lopenpano_ref -L $(PANO_DIR) -lpano_b200 -lpthread \
	  -Wl,-rpath,'$$ORIGIN' -Wl,-rpath,'$$ORIGIN/../../openpano_b200'
