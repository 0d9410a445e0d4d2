#!/bin/bash
# oracle/ref_link_reloc_build.sh — TEST INFRASTRUCTURE.  Links tests/integration/ref_link_reloc_test.cpp and tests/ref_reloc.cpp with the
# objects oracle/ref_link_build.sh compiled (the reference's own translation units, ORBmatcher.cc's symbols weak, and the adapters of
# structure-slam-pointline_b200/host/) and libsslpl_b200.so into oracle/_ref/ref_link_reloc_test (git-ignored, like the rest of
# oracle/_ref/), which tests/test_integration_reloc_gpu.py runs.  build() calls it after ref_link_build.sh where the reference's sources
# are present; elsewhere the binary built there is used.
set -e
HERE="$(cd "$(dirname "$0")" && pwd)"; ROOT="$(cd "$HERE/.." && pwd)"
REF=${SSLPL_REFERENCE_DIR:-/root/reference}
[ -d "$REF/src" ] || { echo "ref_link_reloc_build: $REF absent - keeping the prebuilt binary" >&2; exit 0; }
PKG="$ROOT/structure-slam-pointline_b200"; OUT="$HERE/_ref"; OBJ="$OUT/link_obj"
[ -f "$OBJ/host_matcher_b200.cc.o" ] || { echo "ref_link_reloc_build: run oracle/ref_link_build.sh first" >&2; exit 1; }
CXX=/usr/bin/g++
# the flags of oracle/ref_link_build.sh
FLAGS="-std=c++14 -O2 -ffp-contract=off -fPIC -w -include $PKG/host/ORBextractor.h -I$PKG/host -I$ROOT/include -I$ROOT/oracle/refshim -I$REF/include -I$REF -I$ROOT/oracle"
mkdir -p "$OUT/link_reloc_obj"
$CXX $FLAGS -c "$ROOT/tests/ref_reloc.cpp" -o "$OUT/link_reloc_obj/ref_reloc.o"
$CXX $FLAGS -c "$ROOT/tests/integration/ref_link_reloc_test.cpp" -o "$OUT/link_reloc_obj/main.o"
OBJS=$(ls "$OBJ"/*.o | grep -v '/main\.o$')
$CXX -o "$OUT/ref_link_reloc_test" $OBJS "$OUT/link_reloc_obj/ref_reloc.o" "$OUT/link_reloc_obj/main.o" -L"$PKG" -lsslpl_b200 -L"$ROOT/oracle" -loracle \
     -Wl,-rpath,'$ORIGIN/../../structure-slam-pointline_b200' -Wl,-rpath,'$ORIGIN/..' -lpthread -lm
echo "ref_link_reloc_build: $OUT/ref_link_reloc_test"
