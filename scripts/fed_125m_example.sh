#!/usr/bin/env bash
# MPT-125M federated example: 8 clients, local batch 32, 128 local steps/round, ADOPT + cosine, FedAvg
# (ref: scripts/fed_125m_example.sh:36-103). On an 8-GPU box every GPU hosts one client; the round's
# reduce + server optimizer + broadcast is one fused NVLink kernel (photon.comm_stack.nvl).
LOCAL_BATCH_SIZE=32; LOCAL_STEPS=128; N_CLIENTS=8
TOTAL_STEPS=$((5120 * 256 / LOCAL_BATCH_SIZE)); WARMUP_STEPS=$((100 * 256 / LOCAL_BATCH_SIZE)); N_ROUNDS=$((TOTAL_STEPS / LOCAL_STEPS))
E="llm_config.max_duration=${TOTAL_STEPS}ba llm_config.scheduler.schedulers.lr.t_max=${TOTAL_STEPS}ba"
E="$E llm_config.scheduler.schedulers.lr.t_warmup=${WARMUP_STEPS}ba llm_config.scheduler.schedulers.lr.alpha_f=0.1 llm_config.optimizer.lr=6.0e-4"
E="$E fl.n_rounds=$N_ROUNDS llm_config.local_steps=${LOCAL_STEPS}ba fl.reset_optimizer=false llm_config.save_interval=${LOCAL_STEPS}ba"
E="$E dataset/streams@dataset.train.streams=${N_CLIENTS}_clients dataset/streams@dataset.val.streams=${N_CLIENTS}_clients"
E="$E llm_config.global_train_batch_size=$LOCAL_BATCH_SIZE llm_config.device_train_microbatch_size=auto llm_config.precision=amp_bf16"
E="$E fl.n_total_clients=$N_CLIENTS fl.n_clients_per_round=$N_CLIENTS fl.eval_period=null llm_config.eval_interval=${TOTAL_STEPS}ba"
E="$E photon.checkpoint=false use_wandb=false ~llm_config.loggers.wandb ~llm_config.loggers.tensorboard"
export EXTERNAL_CONFIGS="$E ${EXTERNAL_CONFIGS:-}"
exec bash "$(dirname "${BASH_SOURCE[0]}")/photon_llm.sh" 125M
