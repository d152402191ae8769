# oracle/nes_border.mk -- TEST INFRASTRUCTURE: the UNMODIFIED reference's NES system built with NES_BORDER 1
# (crt_nes.c:64-69, an unguarded #define there) into _ref/, the checkers of libcrt_b200_nes_border.so and
# libcrt_b200_nes_p0_border.so.  Like the scratch-copy recipes of oracle/Makefile: the switch (and, for pattern 0, the
# CRT_CHROMA_PATTERN of crt_nes.h:30) is flipped in a copy in a mktemp dir that is removed again -- no reference source
# ever lands in the repository.  Only where the reference sources lie under $(REF); elsewhere prebuilt files are kept.
#     make -f nes_border.mk
REF     ?= /root/reference
CC      ?= gcc
OUT     := _ref
REFCFLAGS := -O3 -fPIC -w

ifneq ($(wildcard $(REF)/crt_nes.c),)
all: $(OUT)/libref_nes_border.so $(OUT)/libref_nes_p0_border.so
else
all:
	@echo "oracle: $(REF) not present, keeping prebuilt $(OUT)/libref_nes*_border.so"
endif

# PATTERN_nes: the stock chroma pattern 2; PATTERN_nes_p0: pattern 0 (912 samples per line)
PATTERN_nes := 2
PATTERN_nes_p0 := 0

$(OUT)/libref_%_border.so: ref_shim.c
	@mkdir -p $(OUT)
	set -e; T=$$(mktemp -d); cp $(REF)/crt_core.c $(REF)/crt_core.h $(REF)/crt_nes.c $(REF)/crt_nes.h $$T/; \
	sed -i 's/^#define NES_BORDER    0/#define NES_BORDER    1/' $$T/crt_nes.c; \
	sed -i 's/^#define CRT_CHROMA_PATTERN 2/#define CRT_CHROMA_PATTERN $(PATTERN_$*)/' $$T/crt_nes.h; \
	grep -q '^#define NES_BORDER    1' $$T/crt_nes.c; grep -q '^#define CRT_CHROMA_PATTERN $(PATTERN_$*)' $$T/crt_nes.h; \
	$(CC) $(REFCFLAGS) -shared -DCRT_SYSTEM=1 -I$$T -o $@ $$T/crt_core.c $$T/crt_nes.c ref_shim.c; rm -rf $$T

clean:
	rm -f $(OUT)/libref_nes_border.so $(OUT)/libref_nes_p0_border.so

.PHONY: all clean
