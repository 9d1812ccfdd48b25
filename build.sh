#!/bin/bash
# Build libpna_sm90.so in-tree (sm_90a only) and the plain-C oracle.  Same as __graft_entry__.build().
set -e
cd "$(dirname "$0")"
python -c "import __graft_entry__ as g; g.build()"
