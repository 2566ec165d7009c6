#!/usr/bin/env bash
# Copy the UNMODIFIED reference LPIPS module (nnanhuang/S3Gaussian lpipsPyTorch/) into the git-ignored
# oracle/_ref/s3g_ref/lpipsPyTorch/, next to the Python files oracle/build_ref.sh copies, so that tests and
# tools/bench_lpips.py can run the reference module itself (tests/lpips_ref.py patches its weight loading to seeded
# weights).  Nothing here is product code and nothing under oracle/_ref/ is committed.
set -euo pipefail
REF=${REF:-/root/reference}
HERE="$(cd "$(dirname "${BASH_SOURCE[0]}")" && pwd)"
OUT="$HERE/_ref/s3g_ref"
if [ ! -d "$REF/lpipsPyTorch" ]; then
  echo "build_ref_lpips: $REF/lpipsPyTorch not present (GPU box?) - using prebuilt $OUT/lpipsPyTorch if any"; exit 0
fi
mkdir -p "$OUT"
rm -rf "$OUT/lpipsPyTorch"
cp -r "$REF/lpipsPyTorch" "$OUT/lpipsPyTorch"
chmod -R u+w "$OUT/lpipsPyTorch"
echo "build_ref_lpips: ok -> $OUT/lpipsPyTorch"
