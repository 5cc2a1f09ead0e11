# oracle/blend.mk -- TEST INFRASTRUCTURE for hb_blend_cuda (tests/test_blend_gpu.py), on top of oracle/Makefile:
#
#   make -C oracle -f blend.mk blend
#
#   _ref/libhostlogic_blend.so  the product's host filters as in _ref/libhostlogic.so, plus the host blend object
#                               (handbrake_b200/libhb/blend_cuda.c, UNTOUCHED) with its hbcu_blend_* calls redirected to
#                               the plain-C restatement (port/blend_port.c); always built
#   _ref/libhbref_blend.so      the reference's filters as in _ref/libhbref.so, plus the reference's own blend.c (hb_blend)
#                               and its own hb_compute_chroma_smoothing_coefficient, cut out of $(REF)/libhb/common.c (which
#                               as a whole needs FFmpeg, x264 ...); that definition overrides the shim's weak restatement.
#                               Built only where REF names a HandBrake tree: it is needed only to re-record
#                               tests/golden/blend_ref_digests.json (HBCU_RECORD_REF=1) and for tools/bench_blend.py's CPU
#                               column.
# Sources are read where they lie; only symlinks, generated sources and objects are written, all under _ref/.
include Makefile

.PHONY: blend blend-ref
blend: $(OUT)/libhostlogic_blend.so blend-ref

blend-ref:
	@if [ -d $(REF)/libhb ]; then $(MAKE) --no-print-directory -f blend.mk $(OUT)/libhbref_blend.so; \
	 else echo "oracle: no HandBrake tree at $(REF): $(OUT)/libhbref_blend.so (the reference's hb_blend) not built"; fi

# --- the reference's blend -------------------------------------------------------
$(OUT)/src/blend/.staged:
	mkdir -p $(OUT)/src/blend $(OUT)/obj/blend
	ln -sf $(REF)/libhb/blend.c $(OUT)/src/blend/blend.c
	touch $@

$(OUT)/src/blend/ref_chroma_coeff.c: $(OUT)/src/blend/.staged
	{ echo '#include "handbrake/handbrake.h"'; \
	  awk '/^void hb_compute_chroma_smoothing_coefficient\(/ {p = 1} p {print} p && /^}/ {exit}' $(REF)/libhb/common.c; } > $@.tmp
	@grep -q '^void hb_compute_chroma_smoothing_coefficient(' $@.tmp || { echo "oracle: hb_compute_chroma_smoothing_coefficient not found in $(REF)/libhb/common.c" >&2; rm -f $@.tmp; exit 1; }
	mv $@.tmp $@

$(OUT)/obj/blend/blend.o: $(OUT)/src/blend/.staged $(SHIM)/handbrake/handbrake.h
	$(CC) $(CFLAGS) -I$(SHIM) -I$(REF)/libhb -c $(OUT)/src/blend/blend.c -o $@

$(OUT)/obj/blend/ref_chroma_coeff.o: $(OUT)/src/blend/ref_chroma_coeff.c $(SHIM)/handbrake/handbrake.h
	$(CC) $(CFLAGS) -I$(SHIM) -c $< -o $@

$(OUT)/libhbref_blend.so: $(REF_OBJS) $(OUT)/obj/blend/blend.o $(OUT)/obj/blend/ref_chroma_coeff.o $(OUT)/obj/hb_runtime.o \
                          $(OUT)/obj/hb_harness.o $(OUT)/obj/hb_bench.o $(OUT)/obj/ref_registry.o
	$(CC) -shared -o $@ $^ -lm -lpthread

# --- the host blend object over the restatement -------------------------------------
BLEND_HOSTLOGIC := $(HOSTLOGIC_FILTERS) blend_cuda.c
$(OUT)/libhostlogic_blend.so: $(addprefix $(SHIM)/,$(BLEND_HOSTLOGIC)) $(PORT_SRCS) $(SHIM)/hbcu_device_frames.c $(SHIM)/hb_runtime.c \
                              $(SHIM)/hb_harness.c $(SHIM)/hb_harness.h $(SHIM)/handbrake/handbrake.h ../include/hbcu.h hbcu_rename.py
	mkdir -p $(OUT)
	$(CC) -O2 -std=gnu99 -fPIC -shared -w -D__LIBHB__ -pthread $(HBCU_RENAME) -I$(SHIM) -I../include -o $@ \
	    $(addprefix $(SHIM)/,$(BLEND_HOSTLOGIC)) $(PORT_SRCS) $(SHIM)/hbcu_device_frames.c $(SHIM)/hb_runtime.c $(SHIM)/hb_harness.c -lm -lpthread
