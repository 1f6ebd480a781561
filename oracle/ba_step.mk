# oracle/ba_step.mk — builds the checkers of one bundle-adjustment LM iteration (test infrastructure,
# never the product), next to what oracle/Makefile builds:
#
#   make -f ba_step.mk oracle -> oracle/liboracle_ba_step.so              plain-C restatement (orc_ba_step.c)
#   make -f ba_step.mk ref    -> oracle/_ref/libopenpano_ref_ba_step.so   the reference's own TU (refshim/ref_ba_step.cc)
#                                oracle/_ref/ba_step_test                 pano_host.hh's B200BundleAdjusterStep next to
#                                                                         the reference's members (tests/test_gpu_ba_step.py)
# `ref` needs oracle/Makefile's `ref` (libopenpano_ref.so) and openpano_b200/libpano_b200.so first.  Flags are
# oracle/Makefile's parity flags; the reference sources are compiled IN PLACE, outputs go to oracle/_ref/ only.

REF ?= /root/reference
SRC := $(REF)/src
HERE := $(dir $(abspath $(lastword $(MAKEFILE_LIST))))
OUT := $(HERE)_ref
PANO_DIR := $(HERE)../openpano_b200
REF_INC := -I $(SRC) -I $(SRC)/lib -isystem $(SRC)/third-party -I $(HERE)refshim/eigen_stub
CC ?= gcc

.PHONY: all oracle ref
all: oracle ref

oracle: $(HERE)liboracle_ba_step.so
$(HERE)liboracle_ba_step.so: $(HERE)orc_ba_step.c $(HERE)ba_step_api.h $(HERE)oracle_api.h $(HERE)orc_common.h
	$(CC) -std=gnu11 -O2 -ffp-contract=off -msse3 -fPIC -shared -Wall -Wno-unused-function -o $@ $(HERE)orc_ba_step.c -lm

ref:
	@if [ -d "$(SRC)" ]; then $(MAKE) -f $(HERE)ba_step.mk $(OUT)/libopenpano_ref_ba_step.so $(OUT)/ba_step_test; \
	 else echo "oracle/ba_step.mk: $(SRC) not present, keeping prebuilt oracle/_ref/ba_step checkers"; fi

$(OUT)/libopenpano_ref_ba_step.so: $(HERE)refshim/ref_ba_step.cc $(HERE)ba_step_api.h $(HERE)oracle_api.h $(OUT)/libopenpano_ref.so
	g++ -std=c++11 -fPIC -shared -w -DDISABLE_JPEG $(REF_INC) -O2 -ffp-contract=off -msse3 -o $@ $(HERE)refshim/ref_ba_step.cc \
	  -L $(OUT) -lopenpano_ref -Wl,-rpath,'$$ORIGIN'

$(OUT)/ba_step_test: $(HERE)../tests/adaptor/ba_step_test.cc $(PANO_DIR)/host/pano_host.hh $(HERE)../include/pano_b200.h $(HERE)oracle_api.h $(OUT)/libopenpano_ref.so
	g++ -std=c++11 -O1 -ffp-contract=off -msse3 -w -DDISABLE_JPEG $(REF_INC) -I $(HERE)../include -I $(PANO_DIR)/host \
	  -o $@ $< -L $(OUT) -lopenpano_ref -L $(PANO_DIR) -lpano_b200 \
	  -Wl,-rpath,'$$ORIGIN' -Wl,-rpath,'$$ORIGIN/../../openpano_b200'
