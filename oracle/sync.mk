# oracle/sync.mk -- TEST INFRASTRUCTURE: the UNMODIFIED reference built with its decoder's sync searches off
# (CRT_DO_VSYNC / CRT_DO_HSYNC, crt_core.h:71-72, unguarded #defines there) into _ref/, the checkers of the
# libcrt_b200_*_novsync / _nohsync / _nosync libraries and of tests/sync_oracle.py:
#   _ref/libref_<system>_{novsync,nohsync,nosync}.so    every system (CPU builds, cheap)
#   _ref/cli_ref_{ntsc,vhs}_nosync                      crt_main.c with the reference ...
#   _ref/cli_b200_{ntsc,vhs}_nosync                     ... and, unchanged, with libcrt_b200_<system>_nosync.so
#   _ref/video_ref_ntsc_nosync, video_b200_ntsc_nosync  extra/video_convert.c the same two ways (zero_stack_main.c
#                                                       in front, as oracle/Makefile's video_*_ntsc_z)
# Like the scratch-copy recipes of oracle/Makefile: the switches are flipped in a copy in a mktemp dir that is removed
# again -- no reference source ever lands in the repository.  Only where the reference sources lie under $(REF);
# elsewhere prebuilt files are kept.
#     make -f sync.mk
REF     ?= /root/reference
CC      ?= gcc
OUT     := _ref
REFCFLAGS := -O3 -fPIC -w

SYSTEMS  := ntsc vhs nes snes nesrgb template pv1k
SWITCHES := novsync nohsync nosync
SYS_ntsc := 0
SYS_nes := 1
SYS_pv1k := 2
SYS_snes := 3
SYS_template := 4
SYS_vhs := 5
SYS_nesrgb := 6
ENC_ntsc := crt_ntsc.c
ENC_nes := crt_nes.c
ENC_pv1k := crt_pv1k.c
ENC_snes := crt_snes.c
ENC_template := crt_template.c
ENC_vhs := crt_ntscvhs.c
ENC_nesrgb := crt_nesrgb.c
# CRT_DO_VSYNC / CRT_DO_HSYNC of each switch set
V_novsync := 0
H_novsync := 1
V_nohsync := 1
H_nohsync := 0
V_nosync := 0
H_nosync := 0

REFLIBS := $(foreach s,$(SYSTEMS),$(foreach w,$(SWITCHES),$(OUT)/libref_$(s)_$(w).so))
DRIVERS := $(OUT)/cli_ref_ntsc_nosync $(OUT)/cli_b200_ntsc_nosync $(OUT)/cli_ref_vhs_nosync $(OUT)/cli_b200_vhs_nosync \
           $(OUT)/video_ref_ntsc_nosync $(OUT)/video_b200_ntsc_nosync

ifneq ($(wildcard $(REF)/crt_core.h),)
all: $(REFLIBS) $(DRIVERS)
else
all:
	@echo "oracle: $(REF) not present, keeping prebuilt $(OUT)/libref_*_no*sync.so and drivers"
endif

# $(call sys,<target stem>): the system of libref_<system>_<switch> / cli_*_<system>_<switch>; $(call sw,...): the switch
sys = $(firstword $(subst _, ,$(1)))
sw = $(lastword $(subst _, ,$(1)))
# a scratch copy of the reference in $$T with the switches of $(1) flipped in crt_core.h, checked
COPY = T=$$(mktemp -d); cp $(REF)/*.c $(REF)/*.h $$T/; mkdir $$T/extra; cp $(REF)/extra/video_convert.c $$T/extra/; \
	sed -i 's/^\#define CRT_DO_VSYNC    1/\#define CRT_DO_VSYNC    $(V_$(1))/; s/^\#define CRT_DO_HSYNC    1/\#define CRT_DO_HSYNC    $(H_$(1))/' $$T/crt_core.h; \
	grep -q '^\#define CRT_DO_VSYNC    $(V_$(1))' $$T/crt_core.h; grep -q '^\#define CRT_DO_HSYNC    $(H_$(1))' $$T/crt_core.h

$(OUT)/libref_%.so: ref_shim.c
	@mkdir -p $(OUT)
	set -e; $(call COPY,$(call sw,$*)); \
	$(CC) $(REFCFLAGS) -shared -DCRT_SYSTEM=$(SYS_$(call sys,$*)) -I$$T -o $@ $$T/crt_core.c $$T/$(ENC_$(call sys,$*)) ref_shim.c; \
	rm -rf $$T

$(OUT)/cli_ref_%:
	@mkdir -p $(OUT)
	set -e; $(call COPY,$(call sw,$*)); \
	$(CC) -O3 -w -DCRT_SYSTEM=$(SYS_$(call sys,$*)) -I$$T -o $@ $$T/crt_main.c $$T/crt_core.c $$T/$(ENC_$(call sys,$*)) \
		$$T/ppm_rw.c $$T/bmp_rw.c; \
	rm -rf $$T

# drop-in check: the unmodified driver, our header (include/compat/crt_core.h) with the switches given on the command
# line, and the library built with them
B200LIB := ../ntsc-crt_b200/lib
RPATH   := -Wl,-rpath,'$$ORIGIN/../../ntsc-crt_b200/lib'
SWDEFS = -DCRT_DO_VSYNC=$(V_$(1)) -DCRT_DO_HSYNC=$(H_$(1))

$(OUT)/cli_b200_%: $(B200LIB)/libcrt_b200_%.so ../include/crt_b200.h
	@mkdir -p $(OUT)
	$(CC) -O3 -w -DCRT_SYSTEM=$(SYS_$(call sys,$*)) $(call SWDEFS,$(call sw,$*)) -I../include/compat -I$(REF) -o $@ \
		$(REF)/crt_main.c $(REF)/ppm_rw.c $(REF)/bmp_rw.c -L$(B200LIB) -lcrt_b200_$* $(RPATH)

$(OUT)/video_ref_ntsc_nosync: zero_stack_main.c
	@mkdir -p $(OUT)
	set -e; $(call COPY,nosync); \
	$(CC) -O3 -w -DCRT_SYSTEM=0 -Dmain=video_convert_main -I$$T -c -o $$T/video_convert.o $$T/extra/video_convert.c; \
	$(CC) -O3 -w -DCRT_SYSTEM=0 -I$$T -o $@ zero_stack_main.c $$T/video_convert.o $$T/crt_core.c $$T/crt_ntsc.c $$T/bmp_rw.c; \
	rm -rf $$T

$(OUT)/video_b200_ntsc_nosync: zero_stack_main.c $(B200LIB)/libcrt_b200_ntsc_nosync.so ../include/crt_b200.h
	@mkdir -p $(OUT)
	set -e; T=$$(mktemp -d); \
	$(CC) -O3 -w -DCRT_SYSTEM=0 $(call SWDEFS,nosync) -Dmain=video_convert_main -I../include/compat -I$(REF) -c \
		-o $$T/video_convert.o $(REF)/extra/video_convert.c; \
	$(CC) -O3 -w -DCRT_SYSTEM=0 -I$(REF) -o $@ zero_stack_main.c $$T/video_convert.o $(REF)/bmp_rw.c \
		-L$(B200LIB) -lcrt_b200_ntsc_nosync $(RPATH); \
	rm -rf $$T

clean:
	rm -f $(REFLIBS) $(DRIVERS)

.PHONY: all clean
