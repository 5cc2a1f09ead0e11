# oracle/rotate.mk -- TEST INFRASTRUCTURE for the rotate filter (hb_filter_rotate_cuda; tests/test_rotate_gpu.py), on top
# of oracle/format.mk:
#
#   make -C oracle -f rotate.mk rotate
#
#   _ref/libhostlogic_rotate.so  what _ref/libhostlogic_format.so holds (the product's host filters, hb_blend_cuda,
#                                hb_filter_vfr_cuda and hb_filter_format_cuda over the restatements, with two-plane
#                                device frames), plus hb_filter_rotate_cuda (handbrake_b200/libhb/rotate_cuda.c,
#                                UNTOUCHED) over rotate/rotate_port.c, a plain-C restatement of the flips and transposes
#                                behind hbcu_rotate_*.  Always built.
# The reference's side needs nothing new: the chains behind the rotate filter are compared with the reference's filters
# in _ref/libhbref.so (oracle/Makefile) on the rotated input.
include format.mk

.PHONY: rotate
rotate: $(OUT)/libhostlogic_rotate.so

ROTATE_HOSTLOGIC := $(FORMAT_HOSTLOGIC) rotate_cuda.c
ROTATE_PORT_SRCS := $(FORMAT_PORT_SRCS) $(wildcard rotate/*.c)
$(OUT)/libhostlogic_rotate.so: $(addprefix $(SHIM)/,$(ROTATE_HOSTLOGIC)) $(PORT_SRCS) $(wildcard semiplanar/*.c) $(wildcard format/*.c) \
                               $(wildcard rotate/*.c) $(SHIM)/hbcu_device_frames.c $(SHIM)/hb_runtime.c $(SHIM)/hb_harness.c \
                               $(SHIM)/hb_harness.h $(SHIM)/handbrake/handbrake.h ../include/hbcu.h hbcu_rename.py
	mkdir -p $(OUT)
	$(CC) -O2 -std=gnu99 -fPIC -shared -w -D__LIBHB__ -pthread $(HBCU_RENAME) -I$(SHIM) -I../include -o $@ \
	    $(addprefix $(SHIM)/,$(ROTATE_HOSTLOGIC)) $(ROTATE_PORT_SRCS) $(SHIM)/hbcu_device_frames.c $(SHIM)/hb_runtime.c $(SHIM)/hb_harness.c -lm -lpthread
