#!/bin/bash
# oracle/ref_reloc_build.sh — TEST INFRASTRUCTURE.  Compiles tests/ref_reloc.cpp (a C entry point over the reference's own
# ORBmatcher::SearchByProjection(Frame&, KeyFrame*, sAlreadyFound, th, ORBdist)) against the reference's headers and the stand-ins of
# oracle/refshim/, with the flags of oracle/ref_build.sh, into oracle/_ref/libref_reloc.so linked with oracle/_ref/libref.so (git-ignored,
# like the rest of oracle/_ref/).  tests/test_reloc_match_cpu.py loads it.  build() calls it where the reference's sources are present;
# elsewhere the library built there is used.
set -e
HERE="$(cd "$(dirname "$0")" && pwd)"; ROOT="$(cd "$HERE/.." && pwd)"
REF=${SSLPL_REFERENCE_DIR:-/root/reference}
[ -d "$REF/include" ] || { echo "ref_reloc_build: $REF absent - keeping the prebuilt library" >&2; exit 0; }
CXX=${SSLPL_REF_CXX:-/usr/bin/g++}
FLAGS="-std=c++14 -O2 -ffp-contract=off -fno-fast-math -march=x86-64-v3 -fPIC -w -I$HERE/refshim -I$REF/include -I$REF -I$HERE"
$CXX $FLAGS -shared -o "$HERE/_ref/libref_reloc.so" "$ROOT/tests/ref_reloc.cpp" -L"$HERE/_ref" -lref -L"$HERE" -loracle \
     -Wl,-rpath,'$ORIGIN' -Wl,-rpath,'$ORIGIN/..' -Wl,--no-undefined -lpthread
echo "ref_reloc_build: $HERE/_ref/libref_reloc.so"
