# oracle/vfr.mk -- TEST INFRASTRUCTURE for hb_filter_vfr_cuda (tests/test_vfr_gpu.py), on top of oracle/Makefile:
#
#   make -C oracle -f vfr.mk vfr
#
#   _ref/libhostlogic_vfr.so  the product's host filters as in _ref/libhostlogic.so, plus the framerate shaper
#                             (handbrake_b200/libhb/vfr_cuda.c, UNTOUCHED) with its hbcu_motion_metric_* calls redirected
#                             to the plain-C restatement (port/motion_metric_port.c); always built
#   _ref/libhbref_vfr.so      the reference's filters as in _ref/libhbref.so, plus the reference's own vfr.c
#                             (hb_filter_vfr) and motion_metric.c (hb_motion_metric), compiled against the shim.  Built
#                             only where REF names a HandBrake tree: it is needed only to re-record
#                             tests/golden/vfr_ref_digests.json (HBCU_RECORD_REF=1) and for tools/bench_vfr.py's CPU
#                             column.
# Sources are read where they lie; only symlinks and objects are written, all under _ref/.
include Makefile

.PHONY: vfr vfr-ref
vfr: $(OUT)/libhostlogic_vfr.so vfr-ref

vfr-ref:
	@if [ -d $(REF)/libhb ]; then $(MAKE) --no-print-directory -f vfr.mk $(OUT)/libhbref_vfr.so; \
	 else echo "oracle: no HandBrake tree at $(REF): $(OUT)/libhbref_vfr.so (the reference's vfr) not built"; fi

# --- the reference's vfr and motion metric ------------------------------------------
VFR_REF_SRCS := vfr.c motion_metric.c

$(OUT)/src/vfr/.staged:
	mkdir -p $(OUT)/src/vfr $(OUT)/obj/vfr
	for f in $(VFR_REF_SRCS); do ln -sf $(REF)/libhb/$$f $(OUT)/src/vfr/$$f; done
	touch $@

$(OUT)/obj/vfr/%.o: $(OUT)/src/vfr/.staged $(SHIM)/handbrake/handbrake.h $(SHIM)/libavutil/avutil.h
	$(CC) $(CFLAGS) -I$(SHIM) -I$(REF)/libhb -c $(OUT)/src/vfr/$*.c -o $@

$(OUT)/libhbref_vfr.so: $(REF_OBJS) $(addprefix $(OUT)/obj/vfr/,$(VFR_REF_SRCS:.c=.o)) $(OUT)/obj/hb_runtime.o \
                        $(OUT)/obj/hb_harness.o $(OUT)/obj/hb_bench.o $(OUT)/obj/ref_registry.o
	$(CC) -shared -o $@ $^ -lm -lpthread

# --- the host shaper over the restatement ---------------------------------------------
VFR_HOSTLOGIC := $(HOSTLOGIC_FILTERS) vfr_cuda.c
$(OUT)/libhostlogic_vfr.so: $(addprefix $(SHIM)/,$(VFR_HOSTLOGIC)) $(PORT_SRCS) $(SHIM)/hbcu_device_frames.c $(SHIM)/hb_runtime.c \
                            $(SHIM)/hb_harness.c $(SHIM)/hb_harness.h $(SHIM)/handbrake/handbrake.h ../include/hbcu.h hbcu_rename.py
	mkdir -p $(OUT)
	$(CC) -O2 -std=gnu99 -fPIC -shared -w -D__LIBHB__ -pthread $(HBCU_RENAME) -I$(SHIM) -I../include -o $@ \
	    $(addprefix $(SHIM)/,$(VFR_HOSTLOGIC)) $(PORT_SRCS) $(SHIM)/hbcu_device_frames.c $(SHIM)/hb_runtime.c $(SHIM)/hb_harness.c -lm -lpthread
