"""``ops.launch_count()`` counts the kernels each launcher enqueues: for every launcher path, the counter's delta over one call
equals the number of ``pb::`` kernels that ``torch.profiler`` sees on the device (memsets and copies are not kernels and are not
counted). Also: the kernels that opt in to more than 48 KiB of dynamic shared memory run on a second device in the same
process."""
import pytest
import torch

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda", 0)
BF16, F32 = torch.bfloat16, torch.float32


def _rand(*shape, dtype=BF16, dev=DEV, scale=1.0):
    return (torch.randn(*shape, device=dev) * scale).to(dtype)


def _kernels_and_count(fn):
    """(pb:: kernels the profiler saw, launch_count delta) over one call of fn."""
    from torch.autograd import DeviceType
    from torch.profiler import ProfilerActivity, profile

    from photon_b200 import ops

    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        n0 = ops.launch_count()
        fn()
        torch.cuda.synchronize()
        n = ops.launch_count() - n0
    kernels = [e.name for e in prof.events() if e.device_type == DeviceType.CUDA and "pb::" in e.name]
    return kernels, n


# ------------------------------------------------------------------------------------------------ one op per case
def _layernorm_bwd(d, dgamma, dbeta):
    from photon_b200 import ops

    T = 256
    x, dy = _rand(T, d), _rand(T, d)
    gamma = torch.randn(d, device=DEV)
    mean, rstd = torch.zeros(T, device=DEV), torch.ones(T, device=DEV)
    dx = torch.empty_like(x)
    dg = torch.zeros(d, device=DEV) if dgamma else None
    db = torch.zeros(d, device=DEV) if dbeta else None
    return lambda: ops.layernorm_bwd(dy, x, gamma, mean, rstd, None, dx, dg, db)


def _embed_bwd(dwte, dwpe):
    from photon_b200 import ops

    V, S, d = 512, 128, 256
    ids = torch.randint(0, V, (2 * S,), device=DEV)
    dh = _rand(2 * S, d)
    gw = torch.zeros(V, d, device=DEV) if dwte else None
    gp = torch.zeros(S, d, device=DEV) if dwpe else None
    return lambda: ops.embed_bwd(ids, dh, gw, gp, S)


def _gemm():
    from photon_b200 import ops

    a, b, d = _rand(256, 512), _rand(384, 512), torch.empty(256, 384, dtype=BF16, device=DEV)
    return lambda: ops.gemm(a, b, d)


def _gemm_fp8_mn_major():
    from photon_b200 import ops

    M, N, K = 256, 256, 256
    a = _rand(K, M, scale=0.5).to(torch.float8_e4m3fn).view(torch.uint8)
    b = _rand(K, N, scale=0.5).to(torch.float8_e4m3fn).view(torch.uint8)
    d = torch.empty(M, N, dtype=F32, device=DEV)
    meta = torch.ones(3, 2, device=DEV)
    return lambda: ops.gemm_fp8(a, b, d, meta, 0, 1, a_mn=True, b_mn=True, epi=ops.EPI_F32)


def _skinny_gemm(split):
    from photon_b200 import ops

    N, K = (256, 4096) if split else (4096, 64)   # 4 column tiles over 64 k-blocks split K; 64 tiles over 1 k-block do not
    x, w, y = _rand(4, K), _rand(N, K), torch.empty(4, N, dtype=BF16, device=DEV)
    return lambda: ops.skinny_gemm(x, w, y)


def _attention(bwd, doc):
    from photon_b200 import ops

    B, S, H, dh = 2, 256, 2, 64
    qkv = _rand(B, S, 3 * H * dh)
    out, lse = torch.empty(B, S, H * dh, dtype=BF16, device=DEV), torch.empty(B, H, S, device=DEV)
    ds = de = None
    if doc:
        sid = torch.arange(S, device=DEV).div(100, rounding_mode="floor").repeat(B, 1).contiguous()
        ds, de = (torch.empty(B * S, dtype=torch.int32, device=DEV) for _ in range(2))
        ops.doc_bounds(sid, ds, de)
    ops.attention_fwd(qkv, out, lse, H, 0.125, True, None, ds)
    if not bwd:
        return lambda: ops.attention_fwd(qkv, out, lse, H, 0.125, True, None, ds)
    dout, dqkv, delta = _rand(B, S, H * dh), torch.empty_like(qkv), torch.empty_like(lse)
    return lambda: ops.attention_bwd(qkv, out, dout, lse, dqkv, delta, H, 0.125, True, None, ds, de)


def _decode_attention():
    from photon_b200 import ops

    B, H, S, dh = 3, 4, 512, 64
    kc, vc = _rand(B, H, S, dh), _rand(B, H, S, dh)
    q, out = _rand(B, 3 * H * dh), torch.empty(B, H * dh, dtype=BF16, device=DEV)
    pos = torch.tensor([5, 300, 511], dtype=torch.int32, device=DEV)
    return lambda: ops.decode_attention(q, kc, vc, pos, out, H, 0.125)


def _cache_attention(dev=DEV):
    from photon_b200 import ops

    H, S, dh, n = 2, 256, 64, 96
    kc, vc = _rand(2, H, S, dh, dev=dev), _rand(2, H, S, dh, dev=dev)
    qkv, out = _rand(n, 3 * H * dh, dev=dev), torch.zeros(n, H * dh, dtype=BF16, device=dev)
    tiles = ops.cache_tiles([(0, 0, 64, 0), (1, 64, 32, 10)], dev)
    return lambda: ops.cache_attention(qkv, kc, vc, tiles, out, H, 0.125), out


def _cross_entropy(dev=DEV):
    from photon_b200 import ops

    R, V = 64, 4096
    logits = _rand(R, V, dev=dev)
    tgt = torch.randint(0, V, (R,), device=dev)
    stats = torch.zeros(4, dtype=torch.float64, device=dev)
    return lambda: ops.cross_entropy(logits, tgt, 1.0 / R, True, stats)


def _flat_l2_norm():
    from photon_b200 import ops

    x = torch.randn(10_001, device=DEV)
    return lambda: ops.flat_l2_norm(x)


def _fp8_quantize_segments():
    from photon_b200 import ops

    src = _rand(4096)
    dst = torch.empty(4096, dtype=torch.uint8, device=DEV)
    seg = torch.tensor([[0, 1000], [1024, 3072]], dtype=torch.int64, device=DEV)
    meta = torch.ones(3, 2, device=DEV)
    return lambda: ops.fp8_quantize_segments(src, dst, seg, meta, 0)


def _engine_microbatch(precision):
    from photon_b200.models.engine import B200Engine
    from photon_b200.models.mpt import MPTConfig

    cfg = MPTConfig(d_model=256, n_heads=4, n_layers=2, max_seq_len=256, vocab_size=2048)
    eng = B200Engine(cfg, DEV, precision, {"cuda_graph": False}, seed=5)
    ids = torch.randint(0, cfg.vocab_size, (2, cfg.max_seq_len), device=DEV)
    eng.fwd_bwd(ids, float(ids.numel()))   # amp_fp8 calibrates its scales on the first microbatch
    return lambda: eng.fwd_bwd(ids, float(ids.numel()))


CASES = {
    # d = 768 takes the fused LayerNorm backward (one kernel) whenever dgamma or dbeta is given; d = 2048 the split one
    "layernorm_bwd_fused_dgamma_dbeta": (lambda: _layernorm_bwd(768, True, True), 1),
    "layernorm_bwd_fused_dgamma": (lambda: _layernorm_bwd(768, True, False), 1),
    "layernorm_bwd_fused_dbeta": (lambda: _layernorm_bwd(768, False, True), 1),
    "layernorm_bwd_dx_only": (lambda: _layernorm_bwd(768, False, False), 1),
    "layernorm_bwd_split_dgamma_dbeta": (lambda: _layernorm_bwd(2048, True, True), 2),
    "layernorm_bwd_split_dx_only": (lambda: _layernorm_bwd(2048, False, False), 1),
    "embed_bwd_both": (lambda: _embed_bwd(True, True), 2),
    "embed_bwd_wte": (lambda: _embed_bwd(True, False), 1),
    "embed_bwd_wpe": (lambda: _embed_bwd(False, True), 1),
    "embed_bwd_none": (lambda: _embed_bwd(False, False), 0),
    "gemm_bf16": (_gemm, 1),
    "gemm_fp8_mn_major": (_gemm_fp8_mn_major, 3),   # two transposes, then the GEMM
    "skinny_gemm": (lambda: _skinny_gemm(False), 1),
    "skinny_gemm_split_k": (lambda: _skinny_gemm(True), 2),
    "attention_fwd": (lambda: _attention(False, False), 1),
    "attention_fwd_doc": (lambda: _attention(False, True), 1),
    "attention_bwd": (lambda: _attention(True, False), 3),
    "attention_bwd_doc": (lambda: _attention(True, True), 3),
    "decode_attention": (_decode_attention, 2),
    "cache_attention": (lambda: _cache_attention()[0], 1),
    "cross_entropy": (_cross_entropy, 1),
    "flat_l2_norm": (_flat_l2_norm, 2),
    "fp8_quantize_segments": (_fp8_quantize_segments, 2),
    "engine_microbatch_amp_bf16": (lambda: _engine_microbatch("amp_bf16"), None),
    "engine_microbatch_amp_fp8": (lambda: _engine_microbatch("amp_fp8"), None),
}


@pytest.mark.parametrize("case", list(CASES))
def test_launch_count_matches_profiled_kernels(case):
    make, expected = CASES[case]
    fn = make()
    fn()   # warm-up: module loads and shared-memory opt-ins happen outside the profiled call
    kernels, counted = _kernels_and_count(fn)
    assert counted == len(kernels), f"{case}: launch_count says {counted}, the profiler saw {len(kernels)}: {kernels}"
    if expected is not None:
        assert counted == expected, f"{case}: {counted} kernels, expected {expected}: {kernels}"
    else:
        assert counted > 0


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two GPUs")
def test_large_shared_memory_kernels_run_on_a_second_device():
    """The dynamic shared-memory opt-in is an attribute of a kernel on one device: after the kernels have run on device 0, the
    same kernels launched on device 1 in this process must run there too and compute the same results."""
    from photon_b200 import ops

    def run(dev):
        with torch.cuda.device(dev):
            torch.manual_seed(0)
            a, b = _rand(256, 512, dev=dev), _rand(384, 512, dev=dev)
            d = torch.empty(256, 384, dtype=BF16, device=dev)
            ops.gemm(a, b, d)
            qkv = _rand(1, 256, 3 * 2 * 64, dev=dev)
            o, lse = torch.empty(1, 256, 128, dtype=BF16, device=dev), torch.empty(1, 2, 256, device=dev)
            ops.attention_fwd(qkv, o, lse, 2, 0.125, True)
            cache, cache_out = _cache_attention(dev)
            cache()
            x, w = _rand(4, 4096, dev=dev), _rand(256, 4096, dev=dev)
            y = torch.empty(4, 256, dtype=BF16, device=dev)
            ops.skinny_gemm(x, w, y)
            _cross_entropy(dev)()
            torch.cuda.synchronize(dev)
            return [t.cpu() for t in (d, o, cache_out, y)]

    first = run(torch.device("cuda", 0))
    second = run(torch.device("cuda", 1))
    for x0, x1 in zip(first, second):
        assert torch.equal(x0, x1)
