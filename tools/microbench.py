"""Kernel micro-benchmarks (CUDA events on the launching stream, warm-up, L2 flush between timed
launches).  Prints one JSON object per kernel."""
import json, os, subprocess, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from spatialrgpt_b200 import ops

dev = "cuda"
BF = torch.bfloat16
flush_buf = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device=dev)  # > 50 MB L2
peaks = {"hbm_gbs": 3350.0, "bf16_tflops": 989.0}  # H100 SXM data sheet unless MEASURED_PEAKS.json exists
try:
    peaks.update(json.load(open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "MEASURED_PEAKS.json"))))
except Exception:
    pass


def timeit(fn, iters=10, warmup=3, flush=True):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(iters):
        if flush:
            flush_buf.zero_()
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record(); fn(); e.record()
        torch.cuda.synchronize()
        ts.append(s.elapsed_time(e))
    ts.sort()
    return ts[len(ts) // 2], ts[0]


def emit(name, ms, best, bytes_=None, flops=None, **extra):
    r = {"kernel": name, "ms_median": round(ms, 4), "ms_best": round(best, 4)}
    if bytes_ is not None:
        r["GBps"] = round(bytes_ / ms / 1e6, 1); r["frac_hbm"] = round(r["GBps"] / peaks["hbm_gbs"], 3)
    if flops is not None:
        r["TFLOPs"] = round(flops / ms / 1e9, 1); r["frac_tensor"] = round(r["TFLOPs"] / peaks["bf16_tflops"], 3)
    r.update(extra)
    print(json.dumps(r), flush=True)


def rnd(*s):
    return (torch.randn(*s, device=dev) * 0.05).to(BF)


which = sys.argv[1:] or ["gemv", "maskpool", "gemm", "attn", "rowops"]

# the card and its clocks belong beside every number below (nvidia-smi reads them, it changes nothing)
try:
    q = "name,power.limit,clocks.max.sm,clocks.sm"
    smi = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", str(torch.cuda.current_device())],
                         capture_output=True, text=True, timeout=30).stdout.strip()
    print(json.dumps({"gpu": dict(zip(q.split(","), (v.strip() for v in smi.split(","))))}), flush=True)
except (OSError, subprocess.SubprocessError):
    print(json.dumps({"gpu": torch.cuda.get_device_name()}), flush=True)

if "gemv" in which:
    for name, N, K, mode in [("gemv_qkv_rope", 6144, 4096, "qkv"), ("gemv_o", 4096, 4096, "plain"), ("gemv_gateup_swiglu", 28672, 4096, "swiglu"),
                             ("gemv_down", 4096, 14336, "plain"), ("lm_head_argmax", 128259, 4096, "lm")]:
        w, x = rnd(N, K), rnd(K)
        nw = torch.ones(K, dtype=BF, device=dev)
        if mode == "plain":
            y = torch.empty(N, dtype=BF, device=dev); r = rnd(N)
            fn = lambda: ops.gemv(x, w, y, residual=r)
        elif mode == "swiglu":
            y = torch.empty(N // 2, dtype=BF, device=dev)
            fn = lambda: ops.gemv(x, w, y, norm_weight=nw, eps=1e-5, mode=ops.GEMV_SWIGLU)
        elif mode == "qkv":
            from spatialrgpt_b200.config import LlamaDims
            from spatialrgpt_b200.llama_decoder import build_rope_tables
            cos, sin = build_rope_tables(LlamaDims(), 1024, dev)
            pages = torch.zeros(64, 2, 16, 8, 128, dtype=BF, device=dev); pt = torch.arange(64, dtype=torch.int32, device=dev)
            pos = torch.tensor([300], dtype=torch.int32, device=dev); y = torch.empty(4096, dtype=BF, device=dev)
            fn = lambda: ops.gemv(x, w, y, norm_weight=nw, eps=1e-5, mode=ops.GEMV_QKV_ROPE, n_heads=32, n_kv_heads=8, head_dim=128,
                                  cos_tab=cos, sin_tab=sin, pos=pos, kv_pages=pages, page_table=pt, page_size=16)
        else:
            ws = ops.lm_head_workspace(N, dev); ids = torch.zeros(8, dtype=torch.int64, device=dev)
            st = torch.zeros(1, dtype=torch.int32, device=dev); ps = torch.zeros(1, dtype=torch.int32, device=dev)
            def fn():
                st.zero_(); ops.lm_head_argmax(x, w, nw, 1e-5, ws, ids, st, ps)
        ms, best = timeit(fn)
        emit(name, ms, best, bytes_=N * K * 2, N=N, K=K)
    # the same GEMVs over the 12-bit packing (DESIGN.md §3): GBps counts the bytes actually streamed (planes + row metadata)
    for name, N, K, mode in [("gemv_qkv_rope_packed12", 6144, 4096, "qkv"), ("gemv_o_packed12", 4096, 4096, "plain"),
                             ("gemv_gateup_swiglu_packed12", 28672, 4096, "swiglu"), ("gemv_down_packed12", 4096, 14336, "plain"),
                             ("lm_head_argmax_packed12", 128256, 4096, "lm")]:
        w, x = rnd(N, K), rnd(K)
        p, why = ops.pack12(w)
        if p is None:
            raise SystemExit(f"{name}: the matrix stays plain ({why})")
        del w
        nw = torch.ones(K, dtype=BF, device=dev)
        if mode == "plain":
            y = torch.empty(N, dtype=BF, device=dev); r = rnd(N)
            fn = lambda: ops.gemv_packed(x, p, y, residual=r)
        elif mode == "swiglu":
            y = torch.empty(N // 2, dtype=BF, device=dev)
            fn = lambda: ops.gemv_packed(x, p, y, norm_weight=nw, eps=1e-5, mode=ops.GEMV_SWIGLU)
        elif mode == "qkv":
            from spatialrgpt_b200.config import LlamaDims
            from spatialrgpt_b200.llama_decoder import build_rope_tables
            cos, sin = build_rope_tables(LlamaDims(), 1024, dev)
            pages = torch.zeros(64, 2, 16, 8, 128, dtype=BF, device=dev); pt = torch.arange(64, dtype=torch.int32, device=dev)
            pos = torch.tensor([300], dtype=torch.int32, device=dev); y = torch.empty(4096, dtype=BF, device=dev)
            fn = lambda: ops.gemv_packed(x, p, y, norm_weight=nw, eps=1e-5, mode=ops.GEMV_QKV_ROPE, n_heads=32, n_kv_heads=8, head_dim=128,
                                         cos_tab=cos, sin_tab=sin, pos=pos, kv_pages=pages, page_table=pt, page_size=16)
        else:
            ws = ops.lm_head_workspace(N, dev); ids = torch.zeros(8, dtype=torch.int64, device=dev)
            st = torch.zeros(1, dtype=torch.int32, device=dev); ps = torch.zeros(1, dtype=torch.int32, device=dev)
            def fn():
                st.zero_(); ops.lm_head_argmax_packed(x, p, nw, 1e-5, ws, ids, st, ps)
        ms, best = timeit(fn)
        emit(name, ms, best, bytes_=p.nbytes(), N=N, K=K, bf16_equiv_GBps=round(N * K * 2 / ms / 1e6, 1))
    # the layer GEMVs over NF4 planes (4.5 bits per weight; DESIGN.md §3): GBps counts the codes and scales streamed
    for name, N, K, mode in [("gemv_qkv_rope_nf4", 6144, 4096, "qkv"), ("gemv_o_nf4", 4096, 4096, "plain"),
                             ("gemv_gateup_swiglu_nf4", 28672, 4096, "swiglu"), ("gemv_down_nf4", 4096, 14336, "plain")]:
        x = rnd(K)
        codes, scale = ops.nf4_quantize(rnd(N, K))
        p, _ = ops.nf4_planes(codes, scale, ops.nf4_dequantize(codes, scale))
        del codes
        nw = torch.ones(K, dtype=BF, device=dev)
        if mode == "plain":
            y = torch.empty(N, dtype=BF, device=dev); r = rnd(N)
            fn = lambda: ops.gemv_nf4(x, p, y, residual=r)
        elif mode == "swiglu":
            y = torch.empty(N // 2, dtype=BF, device=dev)
            fn = lambda: ops.gemv_nf4(x, p, y, norm_weight=nw, eps=1e-5, mode=ops.GEMV_SWIGLU)
        else:
            from spatialrgpt_b200.config import LlamaDims
            from spatialrgpt_b200.llama_decoder import build_rope_tables
            cos, sin = build_rope_tables(LlamaDims(), 1024, dev)
            pages = torch.zeros(64, 2, 16, 8, 128, dtype=BF, device=dev); pt = torch.arange(64, dtype=torch.int32, device=dev)
            pos = torch.tensor([300], dtype=torch.int32, device=dev); y = torch.empty(4096, dtype=BF, device=dev)
            fn = lambda: ops.gemv_nf4(x, p, y, norm_weight=nw, eps=1e-5, mode=ops.GEMV_QKV_ROPE, n_heads=32, n_kv_heads=8, head_dim=128,
                                      cos_tab=cos, sin_tab=sin, pos=pos, kv_pages=pages, page_table=pt, page_size=16)
        ms, best = timeit(fn)
        emit(name, ms, best, bytes_=p.nbytes(), N=N, K=K, bf16_equiv_GBps=round(N * K * 2 / ms / 1e6, 1))

if "maskpool" in which:
    for (n, side, C, M) in [(1, 128, 1152, 8), (1, 128, 1152, 16), (4, 128, 1152, 4), (32, 128, 1152, 4), (1, 32, 1152, 8), (32, 32, 1152, 4)]:
        L = side * side
        x = rnd(n, L, C)
        masks = (torch.rand(n, M, 448, 448, device=dev) > 0.5).float()
        w = ops.mask_weights(masks, side, ops.ORDER_NESTED if side % 4 == 0 else 0)
        ms, best = timeit(lambda: ops.mask_pool(x, w))
        algo = n * (L * C * 2 + M * L * 2 + M * C * 2)
        emit(f"mask_pool n{n} L{L} C{C} M{M} (dense masks)", ms, best, bytes_=algo)
        boxes = torch.zeros(n, M, 448, 448, device=dev); boxes[:, :, 100:260, 50:300] = 1
        wb = ops.mask_weights(boxes, side, ops.ORDER_NESTED if side % 4 == 0 else 0)
        ms, best = timeit(lambda: ops.mask_pool(x, wb))
        emit(f"mask_pool n{n} L{L} C{C} M{M} (box masks)", ms, best, bytes_=algo)
        ms, best = timeit(lambda: ops.mask_weights(masks, side, ops.ORDER_NESTED if side % 4 == 0 else 0))
        emit(f"mask_weights n{n} M{M} 448->{side}", ms, best, bytes_=n * M * (448 * 448 * 4 + L * 2))
    for n in (1, 32):
        x = rnd(n, 128 * 128, 1152)
        ms, best = timeit(lambda: ops.adaptive_avgpool(x, 128, 27, ops.ORDER_NESTED))
        emit(f"adaptive_avgpool n{n} 128->27 C1152", ms, best, bytes_=n * (128 * 128 * 1152 * 2 + 729 * 1152 * 2))

if "gemm" in which:
    for (M, N, K, epi) in [(2048, 3456, 1152, ops.EPI_BIAS), (2048, 4304, 1152, ops.EPI_BIAS_GELU_TANH), (2048, 1152, 4304, ops.EPI_BIAS_RESIDUAL),
                           (2048, 1152, 1152, ops.EPI_BIAS_RESIDUAL), (8192, 4608, 1152, ops.EPI_BIAS_GELU_ERF),
                           (259, 6144, 4096, ops.EPI_NONE), (259, 28672, 4096, ops.EPI_SWIGLU), (259, 4096, 14336, ops.EPI_BIAS_RESIDUAL),
                           (8288, 6144, 4096, ops.EPI_NONE), (8288, 28672, 4096, ops.EPI_SWIGLU), (8288, 4096, 14336, ops.EPI_BIAS_RESIDUAL),
                           (8192, 8192, 8192, ops.EPI_NONE), (8288, 4096, 4096, ops.EPI_BIAS_RESIDUAL),
                           (65536, 3456, 1152, ops.EPI_BIAS), (65536, 4304, 1152, ops.EPI_BIAS_GELU_TANH), (65536, 1152, 4304, ops.EPI_BIAS_RESIDUAL),
                           (65536, 1152, 1152, ops.EPI_BIAS_RESIDUAL), (65536, 1152, 1152, ops.EPI_NONE), (65536, 1152, 1152, ops.EPI_BIAS),
                           (65536, 1280, 1152, ops.EPI_NONE), (65536, 4304, 1152, ops.EPI_BIAS)]:
        a, w = rnd(M, K), rnd(N, K)
        bias = rnd(N) if epi in (ops.EPI_BIAS, ops.EPI_BIAS_GELU_TANH, ops.EPI_BIAS_GELU_ERF, ops.EPI_BIAS_RESIDUAL) else None
        n_out = N // 2 if epi == ops.EPI_SWIGLU else N
        res = rnd(M, n_out) if epi == ops.EPI_BIAS_RESIDUAL else None
        out = torch.empty(M, n_out, dtype=BF, device=dev)
        ms, best = timeit(lambda: ops.gemm(a, w, bias=bias, residual=res, epilogue=epi, out=out), flush=False)
        emit(f"gemm {M}x{N}x{K} epi{epi}", ms, best, flops=2.0 * M * N * K, bytes_=(M * K + N * K + M * n_out) * 2)

if "cublas" in which:
    # context only: the vendor library (torch.matmul -> cuBLAS) on the short-K SigLIP shapes and one long-K shape, no epilogue
    for (M, N, K) in [(65536, 1152, 1152), (65536, 3456, 1152), (65536, 4304, 1152), (65536, 1152, 4304), (8192, 8192, 8192), (2048, 1152, 1152),
                      (259, 28672, 4096)]:
        a, w = rnd(M, K), rnd(N, K)
        out = torch.empty(M, N, dtype=BF, device=dev)
        ms, best = timeit(lambda: torch.matmul(a, w.t(), out=out), flush=False)
        emit(f"cublas {M}x{N}x{K}", ms, best, flops=2.0 * M * N * K)

if "attn" in which:
    for (B, S, nh, nkv, hd, causal) in [(2, 1024, 16, 16, 72, False), (64, 1024, 16, 16, 72, False), (1, 259, 32, 8, 128, True), (32, 259, 32, 8, 128, True)]:
        qkv = rnd(B * S, (nh + 2 * nkv) * hd)
        qd, kd = nh * hd, nkv * hd
        ms, best = timeit(lambda: ops.attention_prefill(qkv[:, :qd], qkv[:, qd:qd + kd], qkv[:, qd + kd:], B, S, nh, nkv, hd, hd ** -0.5, causal), flush=False)
        fl = 4.0 * B * nh * S * S * hd * (0.5 if causal else 1.0)
        emit(f"attention B{B} S{S} h{nh}/{nkv} hd{hd} causal={causal}", ms, best, flops=fl)

if "rowops" in which:
    x = rnd(2048, 1152); w1 = rnd(1152); b1 = rnd(1152)
    ms, best = timeit(lambda: ops.layernorm(x, w1, b1, 1e-6))
    emit("layernorm 2048x1152", ms, best, bytes_=2048 * 1152 * 4)
    x = rnd(16384, 1152)
    ms, best = timeit(lambda: ops.layernorm(x, w1, b1, 1e-6, act=1))
    emit("layernorm+gelu 16384x1152", ms, best, bytes_=16384 * 1152 * 4)
    x = rnd(259, 4096); w2 = rnd(4096)
    ms, best = timeit(lambda: ops.rmsnorm(x, w2, 1e-5))
    emit("rmsnorm 259x4096", ms, best, bytes_=259 * 4096 * 4)
