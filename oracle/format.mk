# oracle/format.mk -- TEST INFRASTRUCTURE for the pixel-format conversion (hb_filter_format_cuda; tests/test_format_gpu.py),
# on top of oracle/semiplanar.mk:
#
#   make -C oracle -f format.mk format
#
#   _ref/libhostlogic_format.so  what _ref/libhostlogic_semiplanar.so holds (the product's host filters, hb_blend_cuda,
#                                hb_filter_vfr_cuda over the restatements, with two-plane device frames), plus
#                                hb_filter_format_cuda (handbrake_b200/libhb/format_cuda.c, UNTOUCHED) over
#                                format/format_port.c, a plain-C restatement of the four nv12 / p010le <-> yuv420p /
#                                yuv420p10le repacks behind hbcu_format_*.  Always built.
# The reference's side needs nothing new: the chains behind the format filter are compared with the reference's planar
# filters in _ref/libhbref.so (oracle/Makefile).
include semiplanar.mk

.PHONY: format
format: $(OUT)/libhostlogic_format.so

FORMAT_HOSTLOGIC := $(SEMI_HOSTLOGIC) format_cuda.c
FORMAT_PORT_SRCS := $(SEMI_PORT_SRCS) $(wildcard format/*.c)
$(OUT)/libhostlogic_format.so: $(addprefix $(SHIM)/,$(FORMAT_HOSTLOGIC)) $(PORT_SRCS) $(wildcard semiplanar/*.c) $(wildcard format/*.c) \
                               $(SHIM)/hbcu_device_frames.c $(SHIM)/hb_runtime.c $(SHIM)/hb_harness.c $(SHIM)/hb_harness.h \
                               $(SHIM)/handbrake/handbrake.h ../include/hbcu.h hbcu_rename.py
	mkdir -p $(OUT)
	$(CC) -O2 -std=gnu99 -fPIC -shared -w -D__LIBHB__ -pthread $(HBCU_RENAME) -I$(SHIM) -I../include -o $@ \
	    $(addprefix $(SHIM)/,$(FORMAT_HOSTLOGIC)) $(FORMAT_PORT_SRCS) $(SHIM)/hbcu_device_frames.c $(SHIM)/hb_runtime.c $(SHIM)/hb_harness.c -lm -lpthread
