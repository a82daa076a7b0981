#!/usr/bin/env python
"""A/B timing of builds of libKMCUDA.so on the headline shape (run on an H100).  Checker script: it lives
under tests/ because it loads the reference library through oracle/ (not collected by pytest).

    python tests/ab_kernel.py [name=path/to/libKMCUDA.so ...] [--n 8000000] [--env KEY=VAL,...]

Every (library, environment) pair runs in its own process: a parity check of one assignment pass against the
unmodified reference (oracle/_ref) on 100 000 x 256 @ 1024, then CUDA-event timing of the tensor-core kernel and
of the whole step on N x 256 @ 1024 resident samples.  Prints one JSON line per pair.
"""
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def child():
    sys.path.insert(0, ROOT)
    import numpy as np
    import torch
    import kmcuda_b200
    from kmcuda_b200.shard import Shard, assign_once
    n, D, K = int(os.environ.get("AB_N", "8000000")), 256, 1024
    out = {"lib": os.environ.get("AB_NAME"), "env": os.environ.get("AB_ENV", "")}
    # parity on the C1 shape against the reference library
    try:
        from oracle import oracle as O
        import ctypes
        rng = np.random.default_rng(777)
        X = rng.random((100000, D), dtype=np.float32)
        C = X[rng.choice(len(X), K, replace=False)].copy()
        a, _, _, info = assign_once(torch.from_numpy(X).cuda(), torch.from_numpy(C).cuda())
        ref = O.reference_lib()
        A = np.zeros(len(X), np.uint32)
        Cw = C.copy()
        m = ctypes.c_uint32(0)
        rc = ref.kmeans_cuda(3, ctypes.byref(m), 1.0, 0.0, 0, len(X), D, K, 0, 1, -1, 0, 0, X.ctypes.data,
                             Cw.ctypes.data, A.ctypes.data, None)
        out["parity_mismatches"] = int((a.cpu().numpy().astype(np.uint32) != A).sum()) if rc == 0 else "ref rc %d" % rc
        out["parity_rechecked"] = info[1]
        out["parity_overflowed"] = info[2]
    except Exception as e:  # pragma: no cover
        out["parity_error"] = repr(e)[:200]
    g = torch.Generator(device="cuda").manual_seed(777)
    X = torch.rand((n, D), generator=g, device="cuda", dtype=torch.float32)
    C = X[torch.randperm(n, generator=g, device="cuda")[:K]].contiguous()
    sh = Shard(n, D, K)
    a = torch.full((n,), -1, dtype=torch.int32, device="cuda")
    prev = torch.full((n,), -1, dtype=torch.int32, device="cuda")
    ch = torch.zeros(1, dtype=torch.int32, device="cuda")
    for _ in range(3):
        sh.assign(X, C, a, prev, ch)
    torch.cuda.synchronize()
    steps = 10
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        sh.assign(X, C, a, prev, ch)
    e1.record()
    torch.cuda.synchronize()
    kt = sh.kernel_times(steps)
    sums = torch.zeros((K, D), dtype=torch.float32, device="cuda")
    counts = torch.zeros(K, dtype=torch.int32, device="cuda")
    sh.partial_sums(X, a, sums, counts)
    u0, u1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    u0.record()
    for _ in range(5):
        sh.partial_sums(X, a, sums, counts)
    u1.record()
    torch.cuda.synchronize()
    out["partial_sums_ms"] = u0.elapsed_time(u1) / 5
    ab = torch.randint(0, K, (n,), generator=g, device="cuda", dtype=torch.int32)   # balanced clusters
    sh.partial_sums(X, ab, sums, counts)
    u0.record()
    for _ in range(5):
        sh.partial_sums(X, ab, sums, counts)
    u1.record()
    torch.cuda.synchronize()
    out["partial_sums_balanced_ms"] = u0.elapsed_time(u1) / 5
    out["sums_checksum"] = float(sums.double().sum().item())
    tc, rq, ov = sh.last_pass_info()
    out.update({"n": n, "step_ms": e0.elapsed_time(e1) / steps, "kernel_ms": sum(kt) / len(kt), "kernel_ms_min": min(kt),
                "tc": tc, "rechecked": rq, "overflowed": ov, "err": hex(sh.last_error()),
                "tflops_kernel": 2.0 * n * K * D / (sum(kt) / len(kt) * 1e-3) / 1e12,
                "tflops_step": 2.0 * n * K * D / (e0.elapsed_time(e1) / steps * 1e-3) / 1e12})
    print("AB " + json.dumps(out), flush=True)


def main():
    libs, envs, n = [], [""], "8000000"
    args = sys.argv[1:]
    i = 0
    while i < len(args):
        if args[i] == "--n":
            n = args[i + 1]; i += 2
        elif args[i] == "--env":
            envs = args[i + 1].split(";"); i += 2
        else:
            libs.append(args[i]); i += 1
    if not libs:
        libs = ["product=" + os.path.join(ROOT, "kmcuda_b200", "libKMCUDA.so")]
    for spec in libs:
        name, path = spec.split("=", 1)
        for ev in envs:
            env = dict(os.environ, AB_CHILD="1", AB_NAME=name, AB_ENV=ev, AB_N=n, KMCUDA_B200_LIB=os.path.abspath(path))
            for kv in filter(None, ev.split(",")):
                k, v = kv.split("=", 1)
                env[k] = v
            r = subprocess.run([sys.executable, os.path.abspath(__file__)], env=env, stdout=subprocess.PIPE,
                               stderr=subprocess.STDOUT, text=True, timeout=600)
            lines = [ln for ln in r.stdout.splitlines() if ln.startswith("AB ")]
            print(lines[-1] if lines else "AB " + json.dumps({"lib": name, "env": ev, "failed": r.stdout[-600:]}), flush=True)


if __name__ == "__main__":
    child() if os.environ.get("AB_CHILD") == "1" else main()
