#!/usr/bin/env bash
# TEST INFRASTRUCTURE — builds oracle/ref_intersect.cpp and the reference's own intersect.cpp (read in place, not one of build_ref.sh's
# translation units) into oracle/_ref/libtrinity_ref_isect.so, linked against the reference objects of oracle/_ref/libtrinity_ref.so
# (build_ref.sh runs first).  queryexec_ctx.h gets the same generated g++ fix build_ref.sh applies.  Outputs only under oracle/_ref/
# (git-ignored; reused as is where the reference tree is absent).
set -euo pipefail
HERE="$(cd "$(dirname "$0")" && pwd)"
REF="${TRINITY_REFERENCE:-/root/reference}"
OUT="$HERE/_ref"
if [ ! -d "$REF" ]; then
  if [ -f "$OUT/libtrinity_ref_isect.so" ]; then echo "reference absent; using prebuilt $OUT/libtrinity_ref_isect.so"; exit 0; fi
  echo "FATAL: reference tree $REF not found and no prebuilt oracle/_ref/libtrinity_ref_isect.so" >&2; exit 1
fi
[ -f "$OUT/libtrinity_ref.so" ] || { echo "FATAL: run oracle/build_ref.sh first" >&2; exit 1; }
GEN="$OUT/gen_isect"
rm -rf "$GEN"; mkdir -p "$GEN"
python3 - "$REF" "$GEN" <<'PY'
import re, sys
ref, gen = sys.argv[1], sys.argv[2]
src = open(f"{ref}/queryexec_ctx.h").read()
pat = re.compile(r"struct\s*\{\s*(#ifndef USE_BANKS.*?#endif\s*isrc_docid_t maxTrackedDocumentID\{0\}, lastMatchedDocumentID\{0\};)\s*\};", re.S)
new, n = pat.subn(lambda m: m.group(1), src)
assert n == 1, "anonymous-struct patch did not apply exactly once"
open(f"{gen}/queryexec_ctx.h", "w").write(new)
stub = open(f"{ref}/Switch/ext_snappy/snappy-stubs-public.h.in").read()
for k, v in {"${HAVE_SYS_UIO_H_01}": "1", "${PROJECT_VERSION_MAJOR}": "1", "${PROJECT_VERSION_MINOR}": "1", "${PROJECT_VERSION_PATCH}": "7"}.items():
    stub = stub.replace(k, v)
open(f"{gen}/snappy-stubs-public.h", "w").write(stub)
PY
ARCH="${TRINITY_REF_MARCH:-x86-64-v3}"
g++ -std=c++17 -fPIC -fno-rtti -O2 -march=$ARCH -fno-strict-aliasing -DLEAN_SWITCH -D_REENTRANT -w \
  -I"$GEN" -I"$HERE/shim" -I"$REF" -I"$REF/Switch" -I"$REF/Switch/ext_snappy" -I"$REF/Switch/ext/FastPFor/headers" \
  -shared -o "$OUT/libtrinity_ref_isect.so" "$HERE/ref_intersect.cpp" "$REF/intersect.cpp" -L"$OUT" -ltrinity_ref -Wl,-rpath,'$ORIGIN' -lpthread -lz
rm -rf "$GEN"
echo "built $OUT/libtrinity_ref_isect.so"
