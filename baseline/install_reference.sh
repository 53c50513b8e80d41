#!/usr/bin/env bash
# Installs the UNMODIFIED reference package into baseline/_ref (git-ignored).  Usage: install_reference.sh <reference checkout>
# The reference is pure Python; its hard dependencies that are absent offline (librosa, soundfile, sox, onnxruntime,
# transformers==4.57.3) are not installed — bench.py's reference arm imports it through the three probe-only shims of
# oracle/ref_shims.py (SURVEY.md App. B.1) and drives its modules by hand (its HF generate() loop cannot run under
# the installed transformers 5.5.0).  pip builds from a copy, so the checkout may be read-only.
set -euo pipefail
ROOT="$(cd "$(dirname "$0")/.." && pwd)"
SRC="${1:?usage: $0 <reference checkout>}"
[ -d "$SRC/qwen_tts" ] || { echo "no reference at $SRC"; exit 1; }
TMP="$(mktemp -d)"
cp -r "$SRC" "$TMP/ref"
rm -rf "$ROOT/baseline/_ref"
python -m pip install --no-index --no-build-isolation --no-deps --find-links /opt/wheelhouse \
  --target "$ROOT/baseline/_ref" "$TMP/ref"
rm -rf "$TMP"
echo "installed: $(ls "$ROOT/baseline/_ref")"
