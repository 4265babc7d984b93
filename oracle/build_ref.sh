#!/usr/bin/env bash
# TEST INFRASTRUCTURE ONLY — builds the UNMODIFIED reference (hungpham2511/toppra v0.6.2)
# from the checkout named by $TOPPRA_REFERENCE (default /root/reference), where its sources lie, into oracle/_ref/
# (git-ignored).  Used by the tests that run the reference's own classes and files, by bench.py's CPU baseline and to
# regenerate tests/golden (tests/golden/make_golden.py).
#
# Recipe (SURVEY.md §8c):
#   1. stage toppra/ + setup.py + VERSION + README.md into a scratch dir under /tmp
#      (the reference tree is read-only and `build_ext --inplace` writes next to the sources);
#   2. one mechanical shim: cy_seidel_solverwrapper.pyx:8 `ctypedef np.int_t INT_t` does not
#      compile against numpy >= 2 -> `np.int64_t` (the same C type np.int_t had on Linux x86-64);
#   3. `python setup.py build_ext --inplace` (the reference's own flags: -O1);
#   4. install the built package (py + .so) into oracle/_ref/toppra.
# Nothing from the reference is committed to this repository; oracle/_ref/ is in .gitignore.
set -euo pipefail
HERE="$(cd "$(dirname "${BASH_SOURCE[0]}")" && pwd)"
REF="${TOPPRA_REFERENCE:-/root/reference}"
OUT="$HERE/_ref"
if [ ! -d "$REF/toppra" ]; then
  echo "[build_ref] no reference checkout at '$REF' (set TOPPRA_REFERENCE) - keeping $OUT as it is" >&2
  exit 0
fi
SCRATCH="$(mktemp -d /tmp/toppra_ref_build.XXXXXX)"
trap 'rm -rf "$SCRATCH"' EXIT
cp -r "$REF/toppra" "$REF/setup.py" "$REF/VERSION" "$REF/README.md" "$REF/requirements3.txt" "$SCRATCH/"
[ -f "$REF/requirements.txt" ] && cp "$REF/requirements.txt" "$SCRATCH/"
sed -i 's/^ctypedef np.int_t INT_t/ctypedef np.int64_t INT_t/' \
    "$SCRATCH/toppra/solverwrapper/cy_seidel_solverwrapper.pyx"
( cd "$SCRATCH" && python setup.py build_ext --inplace >"$SCRATCH/build.log" 2>&1 ) || {
  tail -n 40 "$SCRATCH/build.log" >&2; exit 1; }
rm -rf "$OUT"; mkdir -p "$OUT"
cp -r "$SCRATCH/toppra" "$OUT/toppra"
find "$OUT" \( -name '*.c' -o -name '*.pyx' -o -name '*.pyc' \) -type f -delete
find "$OUT" -depth -name '__pycache__' -type d -exec rm -rf {} +
echo "[build_ref] reference built into $OUT"
