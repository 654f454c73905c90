# oracle/trim.mk -- TEST INFRASTRUCTURE ONLY (never linked into the product).
#
#   make -f trim.mk ref -> oracle/_ref/libmagickref_trim.so : ref_trim.c against the UNMODIFIED reference archive that
#                                                            oracle/Makefile's `ref` target compiles from source (run
#                                                            that first); skipped without a reference
# The reference's results are stored as digests (tests/golden/trim_digests.json), so the tests need no oracle of their
# own.  Same compiler and flags as oracle/Makefile; every output is git-ignored.

REF      ?= /root/reference
HERE     := $(dir $(abspath $(lastword $(MAKEFILE_LIST))))
OUT      := $(HERE)_ref
CC       := /usr/bin/gcc
REFCFLAGS := -O2 -g0 -fopenmp -fPIC -ffp-contract=off -fexcess-precision=standard -w \
  -DMAGICKCORE_QUANTUM_DEPTH=16 -DMAGICKCORE_HDRI_ENABLE=1 -DMAGICKCORE_CHANNEL_MASK_DEPTH=32 \
  -D_MAGICKLIB_ -DHAVE_CONFIG_H \
  -I$(OUT)/gen -I$(HERE)refconfig -I$(REF)

.PHONY: ref

ifneq ($(wildcard $(REF)/MagickCore/effect.c),)
ref: $(OUT)/libmagickref_trim.so
else
ref:
	@echo "oracle: $(REF) absent - using prebuilt oracle/_ref if present"
endif

$(OUT)/libmagickref_trim.so: $(HERE)ref_trim.c $(HERE)ref_geometry.c $(HERE)ref_harness.c $(OUT)/libMagickCoreRef.a
	$(CC) $(REFCFLAGS) -shared -o $@ $(HERE)ref_trim.c \
	  -Wl,--whole-archive $(OUT)/libMagickCoreRef.a -Wl,--no-whole-archive -lm -lpthread -lgomp
