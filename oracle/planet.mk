# oracle/planet.mk — builds the checkers of the little-planet view, planet() (main.cc:294-331) (test
# infrastructure, never the product), next to what oracle/Makefile builds:
#
#   make -f planet.mk oracle -> oracle/liboracle_planet.so               plain-C restatement (orc_planet.c)
#   make -f planet.mk ref    -> oracle/_ref/libopenpano_ref_planet.so    the reference's own planet() (refshim/ref_planet.cc)
#                               oracle/_ref/planet_test                  pano_host.hh's b200_planet next to the
#                                                                        reference's planet() (tests/test_gpu_planet.py)
# `ref` needs oracle/Makefile's `ref` (libopenpano_ref.so) and openpano_b200/libpano_b200.so first.  Flags are
# oracle/Makefile's parity flags; the reference sources are compiled IN PLACE, outputs go to oracle/_ref/ only.
# main.cc is one TU with the whole CLI: with hidden visibility, one section per function and --gc-sections,
# the linker keeps planet() and what it calls and drops work() / test_*() with the Stitcher code they need;
# --no-undefined makes a symbol that is still missing a build error instead of a load-time one.

REF ?= /root/reference
SRC := $(REF)/src
HERE := $(dir $(abspath $(lastword $(MAKEFILE_LIST))))
OUT := $(HERE)_ref
PANO_DIR := $(HERE)../openpano_b200
REF_INC := -I $(SRC) -I $(SRC)/lib -isystem $(SRC)/third-party -I $(HERE)refshim/eigen_stub
CC ?= gcc

.PHONY: all oracle ref
all: oracle ref

oracle: $(HERE)liboracle_planet.so
$(HERE)liboracle_planet.so: $(HERE)orc_planet.c $(HERE)planet_api.h $(HERE)oracle_api.h $(HERE)orc_common.h
	$(CC) -std=gnu11 -O2 -ffp-contract=off -msse3 -fPIC -shared -Wall -Wno-unused-function -o $@ $(HERE)orc_planet.c -lm

ref:
	@if [ -d "$(SRC)" ]; then $(MAKE) -f $(HERE)planet.mk $(OUT)/libopenpano_ref_planet.so $(OUT)/planet_test; \
	 else echo "oracle/planet.mk: $(SRC) not present, keeping prebuilt oracle/_ref/planet checkers"; fi

$(OUT)/libopenpano_ref_planet.so: $(HERE)refshim/ref_planet.cc $(HERE)planet_api.h $(OUT)/libopenpano_ref.so
	g++ -std=c++11 -fPIC -shared -w -DDISABLE_JPEG $(REF_INC) -O2 -ffp-contract=off -msse3 \
	  -fvisibility=hidden -ffunction-sections -fdata-sections -o $@ $(HERE)refshim/ref_planet.cc \
	  -Wl,--gc-sections -Wl,--no-undefined -L $(OUT) -lopenpano_ref -Wl,-rpath,'$$ORIGIN'

$(OUT)/planet_test: $(HERE)../tests/adaptor/planet_test.cc $(PANO_DIR)/host/pano_host.hh $(HERE)../include/pano_b200.h $(HERE)planet_api.h $(OUT)/libopenpano_ref_planet.so
	g++ -std=c++11 -O1 -ffp-contract=off -msse3 -w -DDISABLE_JPEG $(REF_INC) -I $(HERE)../include -I $(PANO_DIR)/host \
	  -o $@ $< -L $(OUT) -lopenpano_ref_planet -lopenpano_ref -L $(PANO_DIR) -lpano_b200 \
	  -Wl,-rpath,'$$ORIGIN' -Wl,-rpath,'$$ORIGIN/../../openpano_b200'
