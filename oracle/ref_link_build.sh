#!/bin/bash
# oracle/ref_link_build.sh — TEST INFRASTRUCTURE.  Links the reference's own translation units (compiled unmodified, read in
# place from the reference tree, $SSLPL_REFERENCE_DIR) with the adapters of structure-slam-pointline_b200/host/ and libsslpl_b200.so
# into oracle/_ref/ref_link_test (git-ignored, like the rest of oracle/_ref/), which tests/test_integration_gpu.py runs.  build() calls
# it where the reference's sources are present; elsewhere the binary built there is used.
set -e
HERE="$(cd "$(dirname "$0")" && pwd)"; ROOT="$(cd "$HERE/.." && pwd)"
REF=${SSLPL_REFERENCE_DIR:-/root/reference}
[ -d "$REF/src" ] || { echo "ref_link_build: $REF absent - keeping the prebuilt binary" >&2; exit 0; }
PKG="$ROOT/structure-slam-pointline_b200"; OUT="$HERE/_ref"; mkdir -p "$OUT/link_obj"
make -C "$ROOT/oracle" -s; make -C "$PKG/csrc" -s -j8
CXX=/usr/bin/g++
# the adapter's ORBextractor.h replaces the reference's (same include guard): force it in front of every translation unit
FLAGS="-std=c++14 -O2 -ffp-contract=off -fPIC -w -include $PKG/host/ORBextractor.h -I$PKG/host -I$ROOT/include -I$ROOT/oracle/refshim -I$REF/include -I$REF -I$ROOT/oracle"
REFSRC="src/Frame.cc src/KeyFrame.cc src/MapPoint.cc src/MapLine.cpp src/Map.cc src/KeyFrameDatabase.cc src/ORBmatcher.cc src/LSDmatcher.cpp
        Thirdparty/DBoW2/DBoW2/FORB.cpp Thirdparty/DBoW2/DBoW2/BowVector.cpp Thirdparty/DBoW2/DBoW2/FeatureVector.cpp
        Thirdparty/DBoW2/DBoW2/ScoringObject.cpp Thirdparty/DBoW2/DUtils/Random.cpp Thirdparty/DBoW2/DUtils/Timestamp.cpp"
OBJS=""; pids=""
for s in $REFSRC; do o="$OUT/link_obj/ref_$(echo $s | tr '/' '_').o"; OBJS="$OBJS $o"; ( $CXX $FLAGS -c "$REF/$s" -o "$o" ) & pids="$pids $!"; done
for s in ORBextractor.cc ExtractLineSegment_b200.cc matcher_b200.cc bow_b200.cc; do o="$OUT/link_obj/host_$s.o"; OBJS="$OBJS $o"; ( $CXX $FLAGS -c "$PKG/host/$s" -o "$o" ) & pids="$pids $!"; done
o="$OUT/link_obj/minicv.o"; OBJS="$OBJS $o"; ( $CXX $FLAGS -c "$ROOT/oracle/refshim/minicv.cpp" -o "$o" ) & pids="$pids $!"
o="$OUT/link_obj/main.o"; OBJS="$OBJS $o"; ( $CXX $FLAGS -c "$ROOT/tests/integration/ref_link_test.cpp" -o "$o" ) & pids="$pids $!"
for p in $pids; do wait $p; done
# INTEGRATION.md: the bodies the adapters replace are deleted from ORBmatcher.cc / LSDmatcher.cpp; here their symbols are made weak
for s in src_ORBmatcher.cc src_LSDmatcher.cpp src_Frame.cc src_KeyFrame.cc; do objcopy --weaken "$OUT/link_obj/ref_$s.o"; done
$CXX -o "$OUT/ref_link_test" $OBJS -L"$PKG" -lsslpl_b200 -L"$ROOT/oracle" -loracle -Wl,-rpath,'$ORIGIN/../../structure-slam-pointline_b200' -Wl,-rpath,'$ORIGIN/..' -lpthread -lm
echo "ref_link_build: $OUT/ref_link_test"
