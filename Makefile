# sparkflow_b200 developer targets.  GPU targets need a H100 (sm_90a); everything else runs on a CPU box.
PY ?= python
NGPU ?= 8

.PHONY: build test test-gpu smoke bench bench-scale bench-nccl gemm sanitize examples clean

build:            ## nvcc -gencode arch=compute_90a,code=sm_90a -> sparkflow_b200/_C.so, _host.so
	$(PY) tools/build_ext.py

test: build       ## API, formats, oracle, gloo world_size=2 (CPU)
	$(PY) -m pytest tests -q -m "not gpu"

test-gpu: build   ## kernels vs fp32 references, engine vs autograd oracle, multi-GPU
	$(PY) -m pytest tests -q -m gpu

smoke: build
	$(PY) -c "import __graft_entry__ as g; g.smoke()"

bench: build      ## flagship step on one GPU
	$(PY) bench.py --gpus 1 --steps 300 --warmup 30

bench-scale: build
	tools/run_scaling.sh scale 300 30

bench-nccl: build ## the PyTorch + NCCL(+cuBLAS) build of the same semantics
	$(PY) -m torch.distributed.run --nnodes=1 --nproc-per-node $(NGPU) --master-addr 127.0.0.1 bench.py --gpus $(NGPU) --impl nccl

gemm: build       ## one-CTA kernel vs persistent cluster-pair kernel vs cuBLAS
	$(PY) tools/bench_gemm.py

sanitize: build   ## compute-sanitizer over the kernel tests
	tools/sanitize.sh memcheck
	tools/sanitize.sh racecheck "cast_transpose or test_gemm_bias_relu or softmax_xent or im2col"

examples: build
	$(PY) examples/simple_dnn.py && $(PY) examples/cnn_example.py && $(PY) examples/autoencoder_example.py

clean:
	rm -rf build sparkflow_b200/_C.so sparkflow_b200/_host.so .pytest_cache
