#!/usr/bin/env python
"""A/B timing of builds of libKMCUDA.so away from the headline shape (run on an H100; not collected by pytest).

    python tests/ab_shapes.py [name=path/to/libKMCUDA.so ...] [--n 2000000] [--d 128,480] [--k 1024]

For every library and feature count D, a child process runs the assignment pass of a Shard on N x D uniform samples
(seeded on the device) against K of them, and reports the CUDA-event time of `tc_assign_kernel` and of the whole pass,
the re-check / fallback counts and a checksum of the assignments, so builds can be compared output for output.  D = 128
runs the two-K-block pipeline (four B stages, room for two tiles in the A ring), D = 480 the wide one (eight K-blocks,
two B stages).  Prints one JSON line per (library, D).
"""
import hashlib
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def child():
    sys.path.insert(0, ROOT)
    import torch
    from kmcuda_b200.shard import Shard
    n, D, K = int(os.environ["AB_N"]), int(os.environ["AB_D"]), int(os.environ["AB_K"])
    g = torch.Generator(device="cuda").manual_seed(4242)
    X = torch.rand((n, D), generator=g, device="cuda", dtype=torch.float32)
    C = X[torch.randperm(n, generator=g, device="cuda")[:K]].contiguous()
    sh = Shard(n, D, K)
    a = torch.full((n,), -1, dtype=torch.int32, device="cuda")
    prev = torch.full((n,), -1, dtype=torch.int32, device="cuda")
    ch = torch.zeros(1, dtype=torch.int32, device="cuda")
    sh.assign(X, C, a, prev, ch)
    torch.cuda.synchronize()
    digest = hashlib.sha256(a.cpu().numpy().tobytes()).hexdigest()[:16]
    for _ in range(2):
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
    tc, rq, ov = sh.last_pass_info()
    out = {"lib": os.environ.get("AB_NAME"), "n": n, "D": D, "K": K, "assign_sha256": digest,
           "step_ms": e0.elapsed_time(e1) / steps, "kernel_ms": sum(kt) / len(kt), "kernel_ms_min": min(kt),
           "tc": tc, "rechecked": rq, "overflowed": ov, "err": hex(sh.last_error())}
    print("AB " + json.dumps(out), flush=True)


def main():
    libs, n, ds, k = [], "2000000", "128,480", "1024"
    args = sys.argv[1:]
    i = 0
    while i < len(args):
        if args[i] in ("--n", "--d", "--k"):
            n, ds, k = (args[i + 1], ds, k) if args[i] == "--n" else (n, args[i + 1], k) if args[i] == "--d" else \
                (n, ds, args[i + 1])
            i += 2
        else:
            libs.append(args[i]); i += 1
    if not libs:
        libs = ["product=" + os.path.join(ROOT, "kmcuda_b200", "libKMCUDA.so")]
    for d in ds.split(","):
        for spec in libs:
            name, path = spec.split("=", 1)
            env = dict(os.environ, AB_CHILD="1", AB_NAME=name, AB_N=n, AB_D=d, AB_K=k,
                       KMCUDA_B200_LIB=os.path.abspath(path))
            r = subprocess.run([sys.executable, os.path.abspath(__file__)], env=env, stdout=subprocess.PIPE,
                               stderr=subprocess.STDOUT, text=True, timeout=600)
            lines = [ln for ln in r.stdout.splitlines() if ln.startswith("AB ")]
            print(lines[-1] if lines else "AB " + json.dumps({"lib": name, "D": d, "failed": r.stdout[-600:]}), flush=True)


if __name__ == "__main__":
    child() if os.environ.get("AB_CHILD") == "1" else main()
