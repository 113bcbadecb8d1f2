#!/bin/bash
# TEST INFRASTRUCTURE ONLY.  Installs the UNMODIFIED reference (gpauloski/kfac-pytorch, a pure
# Python package) from a reference checkout ($REFERENCE_ROOT) into oracle/_ref/ so that
# `bench.py --impl reference` and the cpu_baseline leg can drive the real
# kfac.preconditioner.KFACPreconditioner on the host cores (oracle/_ref is git-ignored).
# No reference source is copied into the repository history.
set -e
HERE="$(cd "$(dirname "$0")" && pwd)"
REF=${REFERENCE_ROOT:-/root/reference}
if [ ! -d "$REF/kfac" ]; then echo "reference tree not present at $REF: nothing to do"; exit 0; fi
if [ -d "$HERE/_ref/kfac" ]; then echo "oracle/_ref already built"; exit 0; fi
TMP=$(mktemp -d)
cp -r "$REF" "$TMP/src"      # /root/reference is read-only; the build writes an egg-info dir
python -m pip install --quiet --no-index --no-build-isolation --no-deps --find-links /opt/wheelhouse \
    --target "$HERE/_ref" "$TMP/src"
rm -rf "$TMP"
echo "installed reference into $HERE/_ref"
