# oracle/deint.mk -- TEST INFRASTRUCTURE for the Yadif and Bwdif deinterlacers (hb_filter_yadif_cuda,
# hb_filter_bwdif_cuda; tests/test_deinterlace_gpu.py), on top of oracle/rotate.mk:
#
#   make -C oracle -f deint.mk deint
#
#   _ref/libhostlogic_deint.so  what _ref/libhostlogic_rotate.so holds, plus hb_filter_yadif_cuda and
#                               hb_filter_bwdif_cuda (handbrake_b200/libhb/deinterlace_cuda.c, UNTOUCHED) over
#                               deint/deint_port.c, a plain-C restatement of the per-sample arithmetic behind
#                               hbcu_deint_*.  Always built.
# The reference's side needs nothing new: Yadif's interior rows are compared with the reference's decomb (mode=1) in
# _ref/libhbref.so (oracle/Makefile); Bwdif has no counterpart in the reference.
include rotate.mk

.PHONY: deint
deint: $(OUT)/libhostlogic_deint.so

DEINT_HOSTLOGIC := $(ROTATE_HOSTLOGIC) deinterlace_cuda.c
DEINT_PORT_SRCS := $(ROTATE_PORT_SRCS) $(wildcard deint/*.c)
$(OUT)/libhostlogic_deint.so: $(addprefix $(SHIM)/,$(DEINT_HOSTLOGIC)) $(PORT_SRCS) $(wildcard semiplanar/*.c) $(wildcard format/*.c) \
                              $(wildcard rotate/*.c) $(wildcard deint/*.c) $(SHIM)/hbcu_device_frames.c $(SHIM)/hb_runtime.c \
                              $(SHIM)/hb_harness.c $(SHIM)/hb_harness.h $(SHIM)/handbrake/handbrake.h ../include/hbcu.h hbcu_rename.py
	mkdir -p $(OUT)
	$(CC) -O2 -std=gnu99 -fPIC -shared -w -D__LIBHB__ -pthread $(HBCU_RENAME) -I$(SHIM) -I../include -o $@ \
	    $(addprefix $(SHIM)/,$(DEINT_HOSTLOGIC)) $(DEINT_PORT_SRCS) $(SHIM)/hbcu_device_frames.c $(SHIM)/hb_runtime.c $(SHIM)/hb_harness.c -lm -lpthread
