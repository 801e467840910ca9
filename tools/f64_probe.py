"""fp64 GEMM on one H100: the tensor-core (DMMA) kernel against the CUDA-core kernel, TFLOP/s and bit-equality of the two.
    python tools/f64_probe.py [n ...]"""
import os, subprocess, sys, json
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def child(n):
    import torch, laser_b200 as L
    L.init()
    a = torch.rand(n, n, dtype=torch.float64, device="cuda") - 0.5; b = torch.rand(n, n, dtype=torch.float64, device="cuda") - 0.5
    c = torch.empty(n, n, dtype=torch.float64, device="cuda")
    f = lambda: L.gemm_strided(n, n, n, 1.0, a, n, 1, b, n, 1, 0.0, c, n, 1)
    for _ in range(2): f()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    it = 5 if n >= 4096 else 20
    e0.record()
    for _ in range(it): f()
    e1.record(); torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / it
    ref = (a[:64] @ b)
    err = ((c[:64] - ref).abs().max() / ref.abs().max()).item()
    import hashlib
    print(json.dumps(dict(n=n, dmma=os.environ.get("LASER_B200_F64_DMMA", "1"), ms=round(ms, 3), tflops=round(2.0 * n**3 / ms / 1e9, 2),
                          rel_err_vs_torch=err, dmma_launches=int(L.lib().laser_b200_debug_f64_dmma_launches()),
                          sha=hashlib.sha1(c.cpu().numpy().tobytes()).hexdigest()[:16])), flush=True)


if __name__ == "__main__":
    if len(sys.argv) > 2 and sys.argv[1] == "--child":
        child(int(sys.argv[2]))
    else:
        for n in [int(x) for x in sys.argv[1:]] or [2048, 4096, 8192]:
            for dm in ("1", "0"):
                subprocess.run([sys.executable, __file__, "--child", str(n)], env=dict(os.environ, LASER_B200_F64_DMMA=dm))
