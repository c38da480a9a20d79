# oracle/packed.mk — TEST INFRASTRUCTURE: the reference's generic converter steps for audioresample's packed sample
# formats (refshim/refdrv_audio_packed.c) over the reference build of oracle/Makefile:
#
#   _ref/libgstref_packed.so   the reference's audio-quantize.c compiled in place from $(REFROOT), and the driver that
#                              composes unpack -> resample -> quantize -> pack; the unpack / pack functions and the
#                              resampler are those of _ref/libgstref.so, which it links against
#
#   make -C oracle -f packed.mk        (after make -C oracle ref; does nothing where REFROOT is absent)
REFROOT ?= /root/reference
REFBASE := $(REFROOT)/subprojects/gst-plugins-base
REFA    := $(REFBASE)/gst-libs/gst/audio
CC      ?= gcc
REF_CFLAGS := -std=gnu11 -O2 -fPIC -fno-strict-aliasing -w -msse4.1 -DHAVE_CONFIG_H -DDISABLE_ORC -DBUILDING_GST_AUDIO \
              -DHAVE_SSE -DHAVE_SSE2 -DHAVE_SSE41 -Irefshim -I$(REFBASE)/gst-libs -I$(REFA)
OBJDIR := _ref/obj_packed
OBJS := $(OBJDIR)/audio-quantize.o $(OBJDIR)/refdrv_audio_packed.o

.PHONY: all
ifneq ($(wildcard $(REFA)/audio-quantize.c),)
all: _ref/libgstref_packed.so
else
all:
	@echo "oracle/_ref: $(REFROOT) not present; using prebuilt _ref/libgstref_packed.so if any"
endif

$(OBJDIR):
	mkdir -p $(OBJDIR)
$(OBJDIR)/%.o: $(REFA)/%.c | $(OBJDIR)
	$(CC) $(REF_CFLAGS) -c $< -o $@
$(OBJDIR)/%.o: refshim/%.c | $(OBJDIR)
	$(CC) $(REF_CFLAGS) -c $< -o $@
_ref/libgstref_packed.so: $(OBJS) _ref/libgstref.so
	$(CC) -shared -o $@ $(OBJS) -L_ref -l:libgstref.so -Wl,-rpath,'$$ORIGIN' -lm
