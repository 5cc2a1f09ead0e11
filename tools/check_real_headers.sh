#!/bin/bash
# Syntax-only compile of the product's host filter sources against the REAL libhb headers of a HandBrake tree (argument: its libhb directory)
# (not the test shim in handbrake_b200/libhb/handbrake/), backing INTEGRATION.md's claim that they drop into a HandBrake
# tree unchanged.  libav*/jansson are replaced by type-only stubs (tools/real_header_stubs/), project.h by a stand-in
# with every optional feature off.  What is NOT in the real tree and therefore shows up here is exactly the integration
# patch of INTEGRATION.md: the HBCU_DEVICE storage type (passed as a macro) and the three fifo.c hooks
# (hb_shim_set_frame_allocator / hb_shim_set_device_release / hb_shim_set_device_retain).
# usage: tools/check_real_headers.sh [reference libhb dir]      exit 0 = no errors
export LC_ALL=C
REF=${1:?usage: check_real_headers.sh <HandBrake tree>/libhb}
REPO=$(cd "$(dirname "$0")/.." && pwd)
[ -d "$REF/handbrake" ] || { echo "no reference tree at $REF"; exit 2; }
TMP=$(mktemp -d)
# the sources are copied so that #include "handbrake/handbrake.h" cannot find the shim next to them
cp "$REPO"/handbrake_b200/libhb/*_cuda.c "$REPO"/handbrake_b200/libhb/hbcu_*.c "$REPO"/handbrake_b200/libhb/hbcu_*.h "$TMP"/
rc=0
for f in "$TMP"/*.c; do
  out=$(gcc -fsyntax-only -std=gnu99 -Wall -Wno-unused-function -D__LIBHB__ -DHBCU_DEVICE=3 \
        -I "$REPO/tools/real_header_stubs" -I "$REF" -I "$REPO/include" "$f" 2>&1)
  errs=$(echo "$out" | grep -c "error")
  hooks=$(echo "$out" | grep "implicit declaration" | grep -o "'hb_shim_[a-z_]*'" | sort -u | tr '\n' ' ')
  other=$(echo "$out" | grep "warning" | grep -v "hb_shim_" | grep -vc "^$")
  echo "$(basename $f): errors=$errs other_warnings=$other integration_hooks=[${hooks}]"
  [ "$errs" = "0" ] || { echo "$out" | grep error | head -5; rc=1; }
done
rm -rf "$TMP"
exit $rc
