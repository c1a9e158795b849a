# oracle/ref_rgsynth.mk -- TEST INFRASTRUCTURE ONLY.
#
#  make -f ref_rgsynth.mk : compile ref_rgsynth.c with the UNMODIFIED src/share/replaygain_synthesis/replaygain_synthesis.c into
#                           _ref/libFLAC_ref_rgsynth.so with plain gcc -O2, as ref_cli.mk builds the flac tool. Outputs only into _ref/.

REF ?= /root/reference
CC  ?= gcc
OUT := _ref

include Makefile

RGS_SRC   := $(REF)/src/share/replaygain_synthesis/replaygain_synthesis.c
RGS_FLAGS := -O2 -fPIC -shared $(DEFS) -DFLAC__NO_DLL -I$(REF)/include -w

.DEFAULT_GOAL := rgsynth
.PHONY: rgsynth
rgsynth: $(OUT)/libFLAC_ref_rgsynth.so

$(OUT)/libFLAC_ref_rgsynth.so: ref_rgsynth.c $(RGS_SRC)
	@mkdir -p $(OUT)
	$(CC) $(RGS_FLAGS) -o $@ ref_rgsynth.c $(RGS_SRC) -lm
