#!/usr/bin/env bash
# One machine of a cross-host federation (the reference's `flower-supernode`): photon_node.sh SERVER_HOST:PORT
# Connects to the fleet link of a server started with TOPOLOGY=nodes REMOTE_NODES=k (scripts/photon_llm.sh), receives the run's
# config at registration and trains the clients the server hands it on every local GPU (one worker per GPU, DDP / ZeRO inside
# the node). Needs nothing else from the server machine: parameters arrive through the S3 bucket (S3_ENDPOINT_URL, AWS_ACCESS_KEY_ID,
# AWS_SECRET_ACCESS_KEY set here and on the server) or inline in the gRPC messages. PHOTON_FLEET_TOKEN must match the server's.
set -euo pipefail
SERVER=${1:?usage: photon_node.sh SERVER_HOST:PORT}
cd "$(dirname "${BASH_SOURCE[0]}")/.."
# SPMD=1: the whole box joins as ONE node that runs the SPMD runtime inside (one process per GPU, fused NVLink aggregation of the
#         box's clients, one pre-aggregated model per round towards the server) — the shape for multi-box federations of multi-GPU boxes
if [ -n "${SPMD:-}" ]; then
  N=${N_GPUS:-$(python -c "import torch; print(max(1, torch.cuda.device_count()))")}
  exec python -m photon_b200.launch --nproc "$N" --master-port "${BOX_MASTER_PORT:-29600}" -m photon_b200.node -- --server "$SERVER" --spmd ${FLEET_TLS_CA:+--tls-ca "$FLEET_TLS_CA"}
fi
# PER_GPU=1: one node per GPU (each trains its own client at the same time) instead of all GPUs collaborating on one client
exec python -m photon_b200.node --server "$SERVER" ${N_WORKERS:+--n-workers "$N_WORKERS"} ${DEVICES:+--devices "$DEVICES"} ${FLEET_TLS_CA:+--tls-ca "$FLEET_TLS_CA"} ${PER_GPU:+--per-gpu}
