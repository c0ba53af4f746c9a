#!/bin/sh
# Offline install of the UNMODIFIED reference into baseline/_ref (git-ignored).
# The reference ships no setup.py/pyproject.toml, so the
# four modules are copied byte-for-byte into a scratch dir next to a 6-line packaging shim and installed
# from there.  Nothing in ddp.py / model.py / dataset.py / utils.py is edited.
set -e
REPO=$(cd "$(dirname "$0")/.." && pwd)
SRC=${1:?usage: baseline/install_reference.sh <reference checkout> [wheel directory]}
TMP=$(mktemp -d /tmp/ref_pkg.XXXXXX)
cp "$SRC"/ddp.py "$SRC"/model.py "$SRC"/dataset.py "$SRC"/utils.py "$TMP"/
cat > "$TMP/setup.py" <<'PY'
from setuptools import setup
setup(name="pytorch-ddp-template-reference", version="0.0.0",
      py_modules=["ddp", "model", "dataset", "utils"])
PY
rm -rf "$REPO/baseline/_ref"
python -m pip install --no-index --no-build-isolation --no-deps --find-links "${2:-.}" \
    --target "$REPO/baseline/_ref" "$TMP"
for f in ddp.py model.py dataset.py utils.py; do cmp "$SRC/$f" "$REPO/baseline/_ref/$f"; done
echo "reference installed to baseline/_ref (modules byte-identical to $SRC)"
