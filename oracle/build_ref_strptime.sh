#!/bin/sh
# Compiles the reference's strptime_ns translation unit (core/common/Strptime.cpp) IN PLACE from /root/reference (never
# copied into this repo), ahead of oracle/shim on the include path for its StringTools.h, together with
# oracle/ref_strptime_driver.cpp into oracle/_ref/libref_strptime.so.  Without a reference checkout it does nothing.
set -e
cd "$(dirname "$0")"
REF=${LC_REFERENCE:-/root/reference}
[ -f "$REF/core/common/Strptime.cpp" ] || { echo "no reference checkout at $REF"; exit 0; }
mkdir -p _ref
g++ -O2 -std=c++17 -fPIC -shared -Ishim -I"$REF/core" -I"$REF/core/common" \
    "$REF/core/common/Strptime.cpp" ref_strptime_driver.cpp -o _ref/libref_strptime.so
echo "built oracle/_ref/libref_strptime.so"
