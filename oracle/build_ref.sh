#!/usr/bin/env bash
# TEST INFRASTRUCTURE (not product code).
#
# Builds the UNMODIFIED reference (a PreferredAI/cornac checkout, read-only; its
# path in CORNAC_REFERENCE) into oracle/_ref/ so that
#   * tests can validate the C/numpy restatement in oracle/ against the real
#     Cython/OpenMP kernels (cornac/models/bpr/recom_bpr.pyx:208-269,
#     cornac/models/mf/backend_cpu.pyx:35-97, cornac/utils/fast_dot.pyx:40-43),
#   * tests/golden/make_golden.py can generate the committed golden vectors,
#   * bench.py --impl reference can time the reference's own CPU path,
#   * the drop-in models can be exercised through an unchanged cornac.Experiment.
#
# Nothing from the reference is copied into tracked files: oracle/_ref/ is
# git-ignored; a GPU machine without the reference checkout uses the copy built here.
# The reference is a Python/Cython package, so "compiling its few source
# files" means cythonising + g++ on its own setup.py extension list; we build a
# throw-away copy under /tmp because the checkout may be read-only.
#
# Workarounds (SURVEY.md section 8c): a CC wrapper that cannot link -fopenmp
# -> use /usr/bin/gcc; `powerlaw` is a hard import of
# cornac.eval_methods but is not installed -> a 3-line stub module.
set -euo pipefail
HERE="$(cd "$(dirname "${BASH_SOURCE[0]}")" && pwd)"
SRC="${CORNAC_REFERENCE:-/root/reference}"
OUT="$HERE/_ref"
if [ ! -d "$SRC/cornac" ]; then
  echo "[build_ref] $SRC not present - keeping prebuilt $OUT" >&2
  exit 0
fi
if [ -f "$OUT/cornac/models/bpr/recom_bpr.cpython-312-x86_64-linux-gnu.so" ] && [ -z "${FORCE:-}" ]; then
  echo "[build_ref] already built: $OUT" >&2
  exit 0
fi
TMP="$(mktemp -d /tmp/cornac_ref_build.XXXXXX)"
trap 'rm -rf "$TMP"' EXIT
cp -r "$SRC/." "$TMP/"
chmod -R u+w "$TMP"          # the checkout may be read-only; the build writes next to its sources
cd "$TMP"
export CC=/usr/bin/gcc CXX=/usr/bin/g++ LDSHARED="/usr/bin/gcc -shared" LDCXXSHARED="/usr/bin/g++ -shared"
"${PYTHON:-python3}" setup.py build_ext --inplace -j"$(nproc)" > "$TMP/build.log" 2>&1 || { tail -50 "$TMP/build.log"; exit 1; }
rm -rf "$OUT"
mkdir -p "$OUT"
# package only (python sources + freshly built extension modules); no tests/docs/examples
cp -r "$TMP/cornac" "$OUT/cornac"
find "$OUT/cornac" -name '*.cpp' -newer "$SRC/setup.py" -delete 2>/dev/null || true
rm -rf "$OUT/cornac/utils/external"   # vendored boost/eigen headers: build-time only (446k lines)
cp "$HERE/powerlaw_stub.py" "$OUT/powerlaw.py"
( cd "$SRC" && git rev-parse HEAD 2>/dev/null || echo unknown ) > "$OUT/REF_COMMIT"
echo "[build_ref] installed reference into $OUT" >&2
