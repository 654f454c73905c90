# oracle/threshold.mk -- TEST INFRASTRUCTURE ONLY (never linked into the product).
#
#   make -f threshold.mk port -> oracle/libthreshold_oracle.so         : threshold_oracle.c, the plain-C oracle of
#                                                                     AdaptiveThreshold, AutoThreshold, RangeThreshold
#                                                                     and Perceptible (on top of oracle.c)
#   make -f threshold.mk ref  -> oracle/_ref/libmagickref_threshold.so : ref_threshold.c against the UNMODIFIED
#                                                                     reference archive that oracle/Makefile's `ref`
#                                                                     target compiles from source (run that first);
#                                                                     skipped without a reference
# Same compilers and flags as oracle/Makefile; every output is git-ignored.

REF      ?= /root/reference
HERE     := $(dir $(abspath $(lastword $(MAKEFILE_LIST))))
OUT      := $(HERE)_ref
CC       := /usr/bin/gcc
REFCFLAGS := -O2 -g0 -fopenmp -fPIC -ffp-contract=off -fexcess-precision=standard -w \
  -DMAGICKCORE_QUANTUM_DEPTH=16 -DMAGICKCORE_HDRI_ENABLE=1 -DMAGICKCORE_CHANNEL_MASK_DEPTH=32 \
  -D_MAGICKLIB_ -DHAVE_CONFIG_H \
  -I$(OUT)/gen -I$(HERE)refconfig -I$(REF)

.PHONY: all port ref
all: port ref

port: $(HERE)libthreshold_oracle.so
$(HERE)libthreshold_oracle.so: $(HERE)threshold_oracle.c $(HERE)oracle.c $(HERE)oracle.h
	$(CC) -O2 -fPIC -shared -fopenmp -ffp-contract=off -fexcess-precision=standard \
	  -Wall -Wno-unknown-pragmas -o $@ $(HERE)threshold_oracle.c -lm

ifneq ($(wildcard $(REF)/MagickCore/effect.c),)
ref: $(OUT)/libmagickref_threshold.so
else
ref:
	@echo "oracle: $(REF) absent - using prebuilt oracle/_ref if present"
endif

$(OUT)/libmagickref_threshold.so: $(HERE)ref_threshold.c $(HERE)ref_harness.c $(OUT)/libMagickCoreRef.a
	$(CC) $(REFCFLAGS) -shared -o $@ $(HERE)ref_threshold.c \
	  -Wl,--whole-archive $(OUT)/libMagickCoreRef.a -Wl,--no-whole-archive -lm -lpthread -lgomp
