# oracle/pix_formats.mk — builds the checkers of the reference's decoder and encoder layouts (lodepng's RGBA,
# CImg's planes; lib/imgio.cc) (test infrastructure, never the product), next to what oracle/Makefile builds:
#
#   make -f pix_formats.mk oracle -> oracle/liboracle_pix.so              plain-C restatement (orc_pix.c)
#   make -f pix_formats.mk ref    -> oracle/_ref/libopenpano_ref_pix.so   read_img / write_rgb with the reference's own
#                                                                         lodepng and CImg (refshim/ref_pix.cc)
#                                    oracle/_ref/pix_formats_test         pano_host_io.hh's load_pixels / write_mosaic
#                                                                         next to read_img, the reference's detector and
#                                                                         blenders and write_rgb (tests/test_gpu_pixel_formats.py)
# `ref` needs oracle/Makefile's `ref` (libopenpano_ref.so, which holds imgio.cc and lodepng) and
# openpano_b200/libpano_b200.so first.  Flags are oracle/Makefile's parity flags; the reference sources are
# compiled IN PLACE, outputs go to oracle/_ref/ only.

REF ?= /root/reference
SRC := $(REF)/src
HERE := $(dir $(abspath $(lastword $(MAKEFILE_LIST))))
OUT := $(HERE)_ref
PANO_DIR := $(HERE)../openpano_b200
REF_INC := -I $(SRC) -I $(SRC)/lib -isystem $(SRC)/third-party -I $(HERE)refshim/eigen_stub
CC ?= gcc

.PHONY: all oracle ref
all: oracle ref

oracle: $(HERE)liboracle_pix.so
$(HERE)liboracle_pix.so: $(HERE)orc_pix.c $(HERE)pix_api.h
	$(CC) -std=gnu11 -O2 -ffp-contract=off -msse3 -fPIC -shared -Wall -o $@ $(HERE)orc_pix.c

ref:
	@if [ -d "$(SRC)" ]; then $(MAKE) -f $(HERE)pix_formats.mk $(OUT)/libopenpano_ref_pix.so $(OUT)/pix_formats_test; \
	 else echo "oracle/pix_formats.mk: $(SRC) not present, keeping prebuilt oracle/_ref/pix_formats checkers"; fi

$(OUT)/libopenpano_ref_pix.so: $(HERE)refshim/ref_pix.cc $(HERE)pix_api.h $(OUT)/libopenpano_ref.so
	g++ -std=c++11 -fPIC -shared -w -DDISABLE_JPEG $(REF_INC) -O2 -ffp-contract=off -msse3 \
	  -o $@ $(HERE)refshim/ref_pix.cc -Wl,--no-undefined -L $(OUT) -lopenpano_ref -lpthread -Wl,-rpath,'$$ORIGIN'

$(OUT)/pix_formats_test: $(HERE)../tests/adaptor/pix_formats_test.cc $(PANO_DIR)/host/pano_host.hh $(PANO_DIR)/host/pano_host_io.hh $(HERE)../include/pano_b200.h $(OUT)/libopenpano_ref.so
	g++ -std=c++11 -O1 -ffp-contract=off -msse3 -w -DDISABLE_JPEG $(REF_INC) -I $(HERE)../include \
	  -I $(PANO_DIR)/host -o $@ $< -L $(OUT) -lopenpano_ref -L $(PANO_DIR) -lpano_b200 -lpthread \
	  -Wl,-rpath,'$$ORIGIN' -Wl,-rpath,'$$ORIGIN/../../openpano_b200'
