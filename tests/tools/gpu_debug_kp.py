"""Bring-up of the tensor-core kernel-pooling forward: staged parity (each stage in a subprocess) + timing."""
import os, subprocess, sys
ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
STAGES = [(1, 30, 128, 32, 11), (2, 30, 128, 300, 11), (3, 30, 200, 300, 21), (40, 17, 77, 64, 11), (300, 30, 180, 300, 11)]

def stage(i):
    import torch
    from matchmaker_b200 import interaction
    from oracle import interaction_oracle as O
    B, Lq, Ld, D, K = STAGES[i]
    mu, sg = (O.tk_21_kernels() if K == 21 else ([1.0, 0.9, 0.7, 0.5, 0.3, 0.1, -0.1, -0.3, -0.5, -0.7, -0.9], [0.1] * 11))
    mu, sg = torch.tensor(mu), torch.tensor(sg)
    w, alpha = torch.linspace(-0.014, 0.014, K), torch.linspace(0.5, 1.5, K)
    q, d, qm, dm = O.synth_kernel_pool_inputs(B, Lq, Ld, D, seed=7 + i)
    ref, sec = O.kernel_pool_tk(q, d, qm, dm, mu, sg, alpha, w)
    c = [t.cuda() for t in (q, d, qm, dm, mu, sg, w)]
    for impl in ("simt", "tcgen05"):
        out = interaction.kernel_pool(*c, alpha=alpha.cuda(), want_per_kernel=True, impl=impl)
        torch.cuda.synchronize()
        e = (out["score"].cpu() - ref).abs().max().item() / ref.abs().max().item()
        ek = (out["per_kernel"].cpu() - sec["per_kernel"]).abs().max().item() / sec["per_kernel"].abs().max().item()
        print(f"stage {STAGES[i]} {impl}: score rel err {e:.3e} per_kernel rel err {ek:.3e}", flush=True)
        if e > 1e-3: print("  got", out["score"].cpu()[:6].tolist(), "\n  ref", ref[:6].tolist())

def timing():
    import torch
    from matchmaker_b200 import interaction
    from oracle import interaction_oracle as O
    import os
    shapes = [(4096, 30, 200, 300, 21), (4096, 30, 180, 300, 11)]
    if os.environ.get("KP_SHAPES"):
        shapes = [tuple(int(v) for v in sh.split(",")) for sh in os.environ["KP_SHAPES"].split(";")]
    for (B, Lq, Ld, D, K) in shapes:
        mu, sg = (O.tk_21_kernels() if K == 21 else (O.knrm_kernel_mus(11), O.knrm_kernel_sigmas(11)))
        mu, sg = torch.tensor(mu).cuda(), torch.tensor(sg).cuda()
        w, alpha = torch.linspace(-0.014, 0.014, K).cuda(), torch.linspace(0.5, 1.5, K).cuda()
        q, d, qm, dm = [t.cuda() for t in O.synth_kernel_pool_inputs(B, Lq, Ld, D, seed=3)]
        bytes_pair = (Lq + Ld) * D * 4 + (Lq + Ld) * 4 + 4
        for impl in (("tcgen05",) if os.environ.get("KP_SHAPES") else ("tcgen05", "simt")):
            for _ in range(3): interaction.kernel_pool(q, d, qm, dm, mu, sg, w, alpha=alpha, impl=impl)
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(10): interaction.kernel_pool(q, d, qm, dm, mu, sg, w, alpha=alpha, impl=impl)
            e1.record(); torch.cuda.synchronize()
            ms = e0.elapsed_time(e1) / 10
            print(f"timing B={B} Ld={Ld} D={D} K={K} {impl}: {ms:.3f} ms -> {B / ms * 1e3 / 1e6:.2f} M pairs/s, {B * bytes_pair / ms * 1e3 / 1e9:.0f} GB/s", flush=True)

def bwd():
    import torch
    from matchmaker_b200 import autograd, interaction
    from oracle import interaction_oracle as O
    B, Lq, Ld, D, K = 4096, 30, 200, 300, 21
    mu, sg = O.tk_21_kernels()
    mu, sg = torch.tensor(mu).cuda(), torch.tensor(sg).cuda()
    w = torch.linspace(-0.014, 0.014, K).cuda().requires_grad_(True)
    alpha = torch.linspace(0.5, 1.5, K).cuda().requires_grad_(True)
    q, d, qm, dm = [t.cuda() for t in O.synth_kernel_pool_inputs(B, Lq, Ld, D, seed=3)]
    q.requires_grad_(True); d.requires_grad_(True)
    g = torch.randn(B, device="cuda")
    def step():
        s, _ = autograd.kernel_pool(q, d, qm, dm, mu, sg, w, alpha, 1.0)
        s.backward(g)
        q.grad = None; d.grad = None; w.grad = None; alpha.grad = None
    for _ in range(3): step()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(5): step()
    e1.record(); torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / 5
    print(f"TK fwd+bwd B={B}: {ms:.3f} ms per step -> {B / ms * 1e3 / 1e6:.2f} M pairs/s (forward tensor cores + backward FFMA)", flush=True)

if __name__ == "__main__":
    if len(sys.argv) > 1 and sys.argv[1] == "bwd": bwd(); sys.exit(0)
    if len(sys.argv) > 2 and sys.argv[1] == "stage": stage(int(sys.argv[2])); sys.exit(0)
    if len(sys.argv) > 1 and sys.argv[1] == "timing": timing(); sys.exit(0)
    for i in range(len(STAGES)):
        try:
            r = subprocess.run([sys.executable, __file__, "stage", str(i)], timeout=200, capture_output=True, text=True)
            print(r.stdout.strip())
            if r.returncode: print("FAILED", r.stderr[-1500:])
        except subprocess.TimeoutExpired: print("stage", i, "TIMEOUT")
    try:
        r = subprocess.run([sys.executable, __file__, "timing"], timeout=400, capture_output=True, text=True)
        print(r.stdout.strip())
        if r.returncode: print("timing FAILED", r.stderr[-1500:])
    except subprocess.TimeoutExpired: print("timing TIMEOUT")
