#!/usr/bin/env bash
# TEST INFRASTRUCTURE — builds oracle/ref_indexer_payloads.cpp (the reference's indexer fed payloads) into
# oracle/_ref/libtrinity_ref_indexer_payloads.so, linked against the reference objects of
# oracle/_ref/libtrinity_ref.so (SegmentIndexSession, both codecs' IndexSessions; build_ref.sh runs first).  Outputs only under oracle/_ref/
# (git-ignored; reused as is where the reference tree is absent).
set -euo pipefail
HERE="$(cd "$(dirname "$0")" && pwd)"
REF="${TRINITY_REFERENCE:-/root/reference}"
OUT="$HERE/_ref"
if [ ! -d "$REF" ]; then
  if [ -f "$OUT/libtrinity_ref_indexer_payloads.so" ]; then echo "reference absent; using prebuilt $OUT/libtrinity_ref_indexer_payloads.so"; exit 0; fi
  echo "FATAL: reference tree $REF not found and no prebuilt oracle/_ref/libtrinity_ref_indexer_payloads.so" >&2; exit 1
fi
[ -f "$OUT/libtrinity_ref.so" ] || { echo "FATAL: run oracle/build_ref.sh first" >&2; exit 1; }
GEN="$OUT/gen_indexer_payloads"
rm -rf "$GEN"; mkdir -p "$GEN"
python3 - "$REF" "$GEN" <<'PY'
import sys
ref, gen = sys.argv[1], sys.argv[2]
stub = open(f"{ref}/Switch/ext_snappy/snappy-stubs-public.h.in").read()
for k, v in {"${HAVE_SYS_UIO_H_01}": "1", "${PROJECT_VERSION_MAJOR}": "1", "${PROJECT_VERSION_MINOR}": "1", "${PROJECT_VERSION_PATCH}": "7"}.items():
    stub = stub.replace(k, v)
open(f"{gen}/snappy-stubs-public.h", "w").write(stub)
PY
ARCH="${TRINITY_REF_MARCH:-x86-64-v3}"
g++ -std=c++17 -fPIC -fno-rtti -O2 -march=$ARCH -fno-strict-aliasing -DLEAN_SWITCH -D_REENTRANT -w \
  -I"$GEN" -I"$HERE/shim" -I"$REF" -I"$REF/Switch" -I"$REF/Switch/ext_snappy" -I"$REF/Switch/ext/FastPFor/headers" \
  -shared -o "$OUT/libtrinity_ref_indexer_payloads.so" "$HERE/ref_indexer_payloads.cpp" -L"$OUT" -ltrinity_ref -Wl,-rpath,'$ORIGIN' -lpthread -lz
rm -rf "$GEN"
echo "built $OUT/libtrinity_ref_indexer_payloads.so"
