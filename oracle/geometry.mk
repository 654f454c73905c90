# oracle/geometry.mk -- TEST INFRASTRUCTURE ONLY (never linked into the product).
#
#   make -f geometry.mk ref -> oracle/_ref/libmagickref_geometry.so : ref_geometry.c against the UNMODIFIED reference
#                                                                    archive that oracle/Makefile's `ref` target compiles
#                                                                    from source (run that first); skipped without a
#                                                                    reference
# The reference's results are stored as digests (tests/golden/geometry_digests.json), so the tests need no oracle of
# their own.  Same compiler and flags as oracle/Makefile; every output is git-ignored.

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
ref: $(OUT)/libmagickref_geometry.so
else
ref:
	@echo "oracle: $(REF) absent - using prebuilt oracle/_ref if present"
endif

$(OUT)/libmagickref_geometry.so: $(HERE)ref_geometry.c $(HERE)ref_harness.c $(OUT)/libMagickCoreRef.a
	$(CC) $(REFCFLAGS) -shared -o $@ $(HERE)ref_geometry.c \
	  -Wl,--whole-archive $(OUT)/libMagickCoreRef.a -Wl,--no-whole-archive -lm -lpthread -lgomp
