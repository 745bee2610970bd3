# Convenience targets (everything here is a one-liner you can also run by hand; see README.md)
PY ?= python
GPUS ?= 1

.PHONY: build test test-gpu bench bench-scaling smoke clean-shm clean

build:            ## compile csrc/*.cu for sm_90a into photon_b200/_C*.so (works without a GPU)
	$(PY) -m photon_b200.build

test:             ## CPU suite (gloo multi-process, node-manager processes included)
	$(PY) -m pytest tests -q -m "not gpu"

test-gpu:         ## kernel numerics, engine vs torch, NVLink kernels (needs H100s; multi-GPU tests skip on one GPU)
	$(PY) -m pytest tests -q -m gpu

bench:            ## headline metric, one JSON line (GPUS=1|2|4|8)
ifeq ($(GPUS),1)
	$(PY) bench.py --gpus 1 --steps 4 --warmup 3
else
	$(PY) -m torch.distributed.run --nnodes=1 --nproc-per-node $(GPUS) --master-addr 127.0.0.1 bench.py --gpus $(GPUS) --steps 4 --warmup 3
endif

bench-scaling:    ## 1 → 8 GPUs back to back
	bash scripts/bench_scaling.sh

smoke:            ## tiny forward+backward of the flagship model on cuda:0
	$(PY) -c "import __graft_entry__ as g; g.smoke()"

clean-shm:        ## remove /dev/shm segments of crashed runs that have not been touched for 10 minutes
	$(PY) -m photon_b200.clients.utils 600

clean:
	rm -rf build photon_b200/*.so .pytest_cache .hypothesis
	find . -name __pycache__ -type d -prune -exec rm -rf {} +
