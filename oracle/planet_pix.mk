# oracle/planet_pix.mk — builds the checker of the `planet` command from decoded pixels (test infrastructure, never
# the product):
#
#   make -f planet_pix.mk ref -> oracle/_ref/planet_pix_test   pano_host_io.hh's load_pixels / b200_planet /
#                                                              write_mosaic next to the reference's read_img, planet()
#                                                              and write_rgb (tests/test_gpu_planet_pix8.py)
# Needs oracle/Makefile's `ref` (libopenpano_ref.so, which holds imgio.cc and lodepng), oracle/planet.mk's `ref`
# (libopenpano_ref_planet.so, the reference's planet()) and openpano_b200/libpano_b200.so first.  Flags are
# oracle/Makefile's parity flags; outputs go to oracle/_ref/ only.

REF ?= /root/reference
SRC := $(REF)/src
HERE := $(dir $(abspath $(lastword $(MAKEFILE_LIST))))
OUT := $(HERE)_ref
PANO_DIR := $(HERE)../openpano_b200
REF_INC := -I $(SRC) -I $(SRC)/lib -isystem $(SRC)/third-party -I $(HERE)refshim/eigen_stub

.PHONY: ref
ref:
	@if [ -d "$(SRC)" ]; then $(MAKE) -f $(HERE)planet_pix.mk $(OUT)/planet_pix_test; \
	 else echo "oracle/planet_pix.mk: $(SRC) not present, keeping the prebuilt oracle/_ref/planet_pix_test"; fi

$(OUT)/planet_pix_test: $(HERE)../tests/adaptor/planet_pix_test.cc $(PANO_DIR)/host/pano_host.hh $(PANO_DIR)/host/pano_host_io.hh $(HERE)../include/pano_b200.h $(HERE)planet_api.h $(OUT)/libopenpano_ref.so $(OUT)/libopenpano_ref_planet.so
	g++ -std=c++11 -O1 -ffp-contract=off -msse3 -w -DDISABLE_JPEG $(REF_INC) -I $(HERE)../include \
	  -I $(PANO_DIR)/host -o $@ $< -L $(OUT) -lopenpano_ref_planet -lopenpano_ref -L $(PANO_DIR) -lpano_b200 -lpthread \
	  -Wl,-rpath,'$$ORIGIN' -Wl,-rpath,'$$ORIGIN/../../openpano_b200'
