"""Training steps of the classifier on the device (gpdb_train_step_device, Adam) against torch's float32 training of the
same network (cuDNN, TF32 off, torch.optim.Adam) on the same batches, alternating, at B = 64 / 256 / 1 024 images of 15,
3 and 12 channels (ReLU nets). Time per step: CUDA events around `steps` steps after warm-up, median of `reps` windows.
Then, in a separate run, per-kernel times of the device step at B = 256 (15 channels) from torch.profiler. The card's
name, power limit and clocks are read in the same run. Usage: python tools/bench_train.py [out.jsonl]"""
import json
import os
import re
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]


def torch_net(C, w):
    """the network in torch float32 from the .bin arrays (fc1 from k = c + 50 j), as tests/train_reference.py maps it"""
    import torch
    import torch.nn.functional as Fn
    ps = [torch.tensor(np.asarray(a, np.float32)) for a in w]
    fc1 = np.asarray(w[4], np.float32).reshape(144, 50, 500).transpose(2, 1, 0).reshape(500, 7200)
    P = [ps[0].reshape(20, C, 5, 5), ps[1], ps[2].reshape(50, 20, 5, 5), ps[3], torch.tensor(fc1), ps[5],
         ps[6].reshape(500, 2).T, ps[7]]
    P = [p.contiguous().cuda().requires_grad_(True) for p in P]

    def fwd(x):
        a = Fn.max_pool2d(Fn.relu(Fn.conv2d(x, P[0], P[1])), 2, 2)
        a = Fn.max_pool2d(Fn.relu(Fn.conv2d(a, P[2], P[3])), 2, 2)
        return Fn.linear(Fn.relu(Fn.linear(a.reshape(a.shape[0], -1), P[4], P[5])), P[6], P[7])
    return P, fwd


def main():
    import torch

    import train_reference as tr
    from gpd_b200 import lib
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    out = sys.argv[1] if len(sys.argv) > 1 else None
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    rows, steps, reps = [], 10, 5
    for C in (15, 3, 12):
        w = tr.random_net(C, seed=C)
        ctx = lib.Context(lib.default_params(channels=C, relu_after_conv=1))
        ctx.train_begin(lib.train_params(optimizer="adam", lr=1e-4), init=w)
        P, fwd = torch_net(C, w)
        opt = torch.optim.Adam(P, lr=1e-4)
        lossf = torch.nn.CrossEntropyLoss()
        for B in (64, 256, 1024):
            images = torch.from_numpy(tr.random_images(B, C, seed=B)).cuda()
            labels = (torch.arange(B, device="cuda") % 2).to(torch.int32)
            x = images.permute(0, 3, 1, 2).float().contiguous()
            yl = labels.long()

            def dev_step():
                ctx.train_step_tensors(images, labels)

            def torch_step():
                opt.zero_grad(set_to_none=True)
                lossf(fwd(x), yl).backward()
                opt.step()

            ts = {"device": [], "torch": []}
            for f in (dev_step, torch_step):  # warm-up: module load, scratch growth, cuDNN algorithm choice
                for _ in range(3):
                    f()
            torch.cuda.synchronize()
            for _ in range(reps):
                for name, f in (("device", dev_step), ("torch", torch_step)):
                    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    a.record()
                    for _ in range(steps):
                        f()
                    b.record()
                    torch.cuda.synchronize()
                    ts[name].append(a.elapsed_time(b) / steps)
            md, mt = float(np.median(ts["device"])), float(np.median(ts["torch"]))
            row = {"channels": C, "batch": B, "ms_step_device": round(md, 3), "ms_step_torch_fp32": round(mt, 3),
                   "images_per_s_device": round(B / md * 1e3), "images_per_s_torch_fp32": round(B / mt * 1e3),
                   "spread_device_ms": [round(min(ts["device"]), 3), round(max(ts["device"]), 3)],
                   "spread_torch_ms": [round(min(ts["torch"]), 3), round(max(ts["torch"]), 3)], "gpu": gpu}
            print(json.dumps(row), flush=True)
            rows.append(row)
        ctx.close()
    # per-kernel times, a separate run under the profiler
    C, B = 15, 256
    ctx = lib.Context(lib.default_params(channels=C, relu_after_conv=1))
    ctx.train_begin(lib.train_params(optimizer="adam", lr=1e-4), init=tr.random_net(C, seed=C))
    images = torch.from_numpy(tr.random_images(B, C, seed=B)).cuda()
    labels = (torch.arange(B, device="cuda") % 2).to(torch.int32)
    for _ in range(3):
        ctx.train_step_tensors(images, labels)
    torch.cuda.synchronize()
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(5):
            ctx.train_step_tensors(images, labels)
        torch.cuda.synchronize()
    kern = {}
    for e in prof.key_averages():
        if e.device_type.name == "CUDA" and e.count:
            m = re.search(r"\b(k_[a-z0-9_]+)", e.key)
            name = m.group(1) if m else e.key[:48]
            kern[name] = kern.get(name, 0.0) + e.self_device_time_total / 5 / 1e3
    row = {"profile": f"{C} channels, B = {B}, ms per step", "kernels": {k: round(v, 3) for k, v in
                                                                         sorted(kern.items(), key=lambda kv: -kv[1])},
           "gpu": gpu}
    print(json.dumps(row), flush=True)
    rows.append(row)
    if out:
        with open(out, "w") as f:
            f.write("".join(json.dumps(r) + "\n" for r in rows))


if __name__ == "__main__":
    main()
