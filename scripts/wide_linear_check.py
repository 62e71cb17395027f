"""the wide wgmma linear kernel (dense_tc.cu, tcx) against fp64 and against the library GEMM it replaces: error and time"""
import os, sys, torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import gnnb200 as gnn
lib = gnn._lib.lib


def run(N, K, Nout, relu=0, bias=True, reps=5):
    gen = torch.Generator(device="cuda").manual_seed(N + K)
    x = torch.randn(N, K, device="cuda", generator=gen)
    W = torch.randn(Nout, K, device="cuda", generator=gen) / K ** 0.5
    b = torch.randn(Nout, device="cuda", generator=gen) if bias else None
    y = torch.empty(N, Nout, device="cuda")
    out = {}
    for name, on in (("wgmma", 1), ("library", 0)):
        lib.gnnb_dense_set_tensor_core_kernel(on)
        call = lambda: gnn._lib.check(lib.gnnb_linear(x.data_ptr(), W.data_ptr(), None if b is None else b.data_ptr(), relu, N, K, Nout, y.data_ptr(), None))
        call(); call()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(reps):
            call()
        e1.record(); torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / reps
        m = min(N, 20000)
        ref = x[:m].double() @ W.double().t() + (0 if b is None else b.double())
        if relu:
            ref = ref.clamp(min=0)
        err = float((y[:m].double() - ref).norm() / ref.norm())
        tail = float((y[-m:].double() - (lambda r: r.clamp(min=0) if relu else r)(x[-m:].double() @ W.double().t() + (0 if b is None else b.double()))).norm() / ref.norm())
        out[name] = (ms, err, tail)
    lib.gnnb_dense_set_tensor_core_kernel(1)
    tf = 2.0 * N * K * Nout / 1e12
    print(f"N={N} K={K} Nout={Nout}: " + "  ".join(f"{k}: {v[0]:.3f} ms ({tf / v[0] * 1e3:.0f} TFLOP/s fp32-equivalent) err {v[1]:.2e}/{v[2]:.2e}" for k, v in out.items()),
          "tc_error", lib.gnnb_dense_tc_error(), flush=True)


run(5000, 64, 256)
run(40000, 512, 512, relu=1)
run(300000, 256, 256)
run(2_000_000, 512, 512, bias=False, reps=3)
run(12_500_000, 256, 256, relu=1, reps=3)
run(2_000_000, 512, 128, reps=3)
