#!/usr/bin/env bash
# Build the sm_90a extension in-tree (the only "install" step; no network needed).
# ref counterpart: scripts/install_env.sh (poetry + flash-attn build) — nothing of that is required here.
set -euo pipefail
cd "$(dirname "${BASH_SOURCE[0]}")/.."
python -m photon_b200.build "$@"
python -c "import photon_b200._C as C; print('photon_b200._C ok:', len([x for x in dir(C) if not x.startswith('_')]), 'symbols')"
