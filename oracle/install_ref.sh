#!/bin/bash
# Puts the UNMODIFIED reference tree where bench.py's reference-GPU leg (BASELINE.md §4: the denominator of the ">= 6x the
# reference's own cuDNN-backed GPU images/sec" target) can import it.
#
# The reference is a plain script tree (train.py, models/, base/, utils/, ...): it has no setup.py / pyproject.toml, so
#   python -m pip install --no-index --no-build-isolation --target oracle/_ref <reference checkout>
# fails with "neither 'setup.py' nor 'pyproject.toml' found" (recorded in DESIGN.md).  "Installing" it therefore means
# putting the tree on the import path: this recipe packs the Python sources, untouched, into ONE archive,
# oracle/_ref/reference.zip (Python imports packages straight from a zip) — git-ignored (never part of the repo's
# history), a build product like the .so.  Nothing here is product code, and nothing is unpacked into the repo.
# Without a reference checkout the recipe keeps whatever oracle/_ref holds and bench.py's leg uses the oracle port.
set -e
HERE="$(cd "$(dirname "$0")" && pwd)"
SRC="${1:-/root/reference}"
DST="$HERE/_ref"
if [ ! -d "$SRC/models" ]; then
  echo "install_ref: $SRC not present: keeping $DST as it is" >&2
  exit 0
fi
rm -rf "$DST"
mkdir -p "$DST"
python - "$SRC" "$DST/reference.zip" <<'PY'
import os, sys, zipfile
src, dst = sys.argv[1], sys.argv[2]
with zipfile.ZipFile(dst, "w", zipfile.ZIP_DEFLATED) as z:
    for d in ("models", "base", "utils", "dataloaders"):
        for root, _, files in os.walk(os.path.join(src, d)):
            for f in files:
                if f.endswith(".py"):
                    p = os.path.join(root, f)
                    z.write(p, os.path.relpath(p, src))
    for f in ("train.py", "trainer.py", "inference.py", "config.json"):
        z.write(os.path.join(src, f), f)
print("install_ref: reference tree ->", dst)
PY
( cd "$SRC" && git rev-parse HEAD 2>/dev/null || echo unknown ) > "$DST/REFERENCE_COMMIT"
