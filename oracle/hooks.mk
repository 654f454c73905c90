# oracle/hooks.mk -- TEST INFRASTRUCTURE ONLY (never linked into the product).
#
#   make -f hooks.mk port -> oracle/libhooks_oracle.so           : hooks_oracle.c, the plain-C oracle of Despeckle,
#                                                                   LocalContrast and WaveletDenoise
#   make -f hooks.mk ref  -> oracle/_ref/libmagickref_hooks.so    : ref_hooks.c against the UNMODIFIED reference archive
#                                                                   that oracle/Makefile's `ref` target compiles from
#                                                                   source (run that first); skipped without a reference
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

port: $(HERE)libhooks_oracle.so
$(HERE)libhooks_oracle.so: $(HERE)hooks_oracle.c
	$(CC) -O2 -fPIC -shared -fopenmp -ffp-contract=off -fexcess-precision=standard \
	  -Wall -Wno-unknown-pragmas -o $@ $< -lm

ifneq ($(wildcard $(REF)/MagickCore/effect.c),)
ref: $(OUT)/libmagickref_hooks.so
else
ref:
	@echo "oracle: $(REF) absent - using prebuilt oracle/_ref if present"
endif

$(OUT)/libmagickref_hooks.so: $(HERE)ref_hooks.c $(OUT)/libMagickCoreRef.a
	$(CC) $(REFCFLAGS) -shared -o $@ $(HERE)ref_hooks.c \
	  -Wl,--whole-archive $(OUT)/libMagickCoreRef.a -Wl,--no-whole-archive -lm -lpthread -lgomp
