#!/bin/bash
# Before a GPU run: rebuild everything and check that every library loads with every symbol the bindings declare
# (a stale .so fails here instead of on the GPU).
set -e
cd "$(dirname "$0")/.."
make -s -C ntsc-crt_b200/csrc -j8 all > /dev/null
make -s -C oracle all > /dev/null
make -s -C tools all > /dev/null
python - <<'P'
import pkgload; pkgload.load()
from ntsc_crt_b200 import capi
for v in capi.ALL_VARIANTS:
    capi.load(v)
print("preflight: %d libraries load with all declared symbols" % len(capi.ALL_VARIANTS))
P
