# oracle/semiplanar.mk -- TEST INFRASTRUCTURE for semi-planar frames (NV12, P010, P016; tests/test_blend_semiplanar_gpu.py),
# on top of oracle/Makefile:
#
#   make -C oracle -f semiplanar.mk semiplanar
#
#   _ref/libhostlogic_semiplanar.so  the product's host filters as in _ref/libhostlogic.so, plus hb_blend_cuda and
#                                    hb_filter_vfr_cuda (handbrake_b200/libhb/blend_cuda.c, vfr_cuda.c, UNTOUCHED), over
#                                    the restatements of port/ with two of them extended to semi-planar frames:
#                                    semiplanar/hostlogic_frames_semiplanar.c (two-plane device frames) in place of
#                                    port/hostlogic_frames.c, semiplanar/blend_semiplanar_port.c (blend.c's *bi*
#                                    functions) in place of port/blend_port.c; each compiles the file it extends.
#                                    Always built.
# The reference's side needs nothing new: _ref/libhbref_blend.so and _ref/libhbref_vfr.so (blend.mk, vfr.mk) already
# hold blend.c and vfr.c, which take semi-planar frames as they are.
include Makefile

.PHONY: semiplanar
semiplanar: $(OUT)/libhostlogic_semiplanar.so

SEMI_HOSTLOGIC := $(HOSTLOGIC_FILTERS) blend_cuda.c vfr_cuda.c
SEMI_PORT_SRCS := $(filter-out port/blend_port.c port/hostlogic_frames.c,$(PORT_SRCS)) $(wildcard semiplanar/*.c)
$(OUT)/libhostlogic_semiplanar.so: $(addprefix $(SHIM)/,$(SEMI_HOSTLOGIC)) $(PORT_SRCS) $(wildcard semiplanar/*.c) \
                                   $(SHIM)/hbcu_device_frames.c $(SHIM)/hb_runtime.c $(SHIM)/hb_harness.c $(SHIM)/hb_harness.h \
                                   $(SHIM)/handbrake/handbrake.h ../include/hbcu.h hbcu_rename.py
	mkdir -p $(OUT)
	$(CC) -O2 -std=gnu99 -fPIC -shared -w -D__LIBHB__ -pthread $(HBCU_RENAME) -I$(SHIM) -I../include -o $@ \
	    $(addprefix $(SHIM)/,$(SEMI_HOSTLOGIC)) $(SEMI_PORT_SRCS) $(SHIM)/hbcu_device_frames.c $(SHIM)/hb_runtime.c $(SHIM)/hb_harness.c -lm -lpthread
