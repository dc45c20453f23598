"""Per-op device times of one forward pass, measured in one process: build the network, warm it up, time 3 forwards
under torch.profiler (CUDA activities) and join the dcr:: kernel records to the op list (net.meta).  Prints, per op,
M, N, K, the time, the achieved TFLOP/s and GB/s from the algorithmic FLOPs and bytes, the share of the data-sheet
bound (max(FLOPs / 989 TFLOP/s, bytes / 3.35 TB/s) over the measured time: H100 SXM dense bf16 and HBM3) and the
share of the forward; then totals per kernel family.  The card's name and power limit head the table.
usage: python tools/layer_profile.py <sscd|vit|inception> <batch> [--json out.json]"""
import argparse, json, os, re, subprocess, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

PEAK_FLOPS = 989e12   # H100 SXM data sheet, dense bf16
PEAK_BYTES = 3.35e12  # H100 SXM data sheet, HBM3


def describe(meta, batch):
    out = []
    for kind, a in meta:
        if kind == 1:
            h, w, c, n, kh, kw, st, ph, pw = a[2], a[3], a[4], a[6], a[7], a[8], a[9], a[10], a[11]
            ho, wo = (h + 2 * ph - kh) // st + 1, (w + 2 * pw - kw) // st + 1
            m = batch * ho * wo
            k = kh * kw * c
            byt = 2 * (batch * h * w * c + m * n + (m * n if a[14] >= 0 else 0)) + 2 * n * k
            out.append(dict(op="conv", M=m, N=n, K=k, kh=kh, kw=kw, stride=st, flops=2.0 * m * n * k, bytes=byt))
        else:
            names = {0: "im2col_u8", 10: "stem_s2d", 2: "maxpool", 3: "avgpool", 4: "gem", 5: "gap", 6: "layernorm", 7: "tokens", 8: "attention", 9: "l2norm", 11: "embed", 12: "stem_rows", 13: "stem_conv"}
            out.append(dict(op=names.get(kind, str(kind)), M=0, N=0, K=0, flops=0.0, bytes=0))
    return out


def family(name):
    """kernel function name without namespace and template arguments: gemm_bf16_kernel, conv3x3_halo_kernel, ..."""
    return short(name).split("<")[0]


def short(name):
    """kernel name without return type, namespaces and parameter list: gemm_bf16_kernel<128, false, 2>"""
    name = name.replace("(anonymous namespace)::", "").replace("(int)", "").replace("void ", "")
    return re.sub(r"\(.*", "", name).split("::")[-1].strip()


def join(ops, kernels):
    """kernels: [(name, us)] of ONE forward, in launch order -> one row per launch (fused pairs take two ops)"""
    rows, oi = [], 0
    for name, us in kernels:
        o = dict(ops[oi])
        compact = name.replace("(int)", "")
        if "expand_reduce_kernel<0>" in compact:
            o["op"] = "conv3(x3)"                               # expansion-only variant of the fused kernel (in-place residual)
        elif "expand_reduce_kernel" in name:                 # conv3 (+residual) fused with the next block's conv1
            o2 = ops[oi + 1]
            # the expanded activation is written once and never re-read: drop its read from the second conv's bytes
            o = dict(op="conv3+conv1", M=o["M"], N=o["N"], K=o["K"], flops=o["flops"] + o2["flops"],
                     bytes=o["bytes"] + o2["bytes"] - 2 * o["M"] * o["N"])
            oi += 1
        oi += 1
        o["us"], o["kernel"], o["family"] = us, short(name), family(name)
        rows.append(o)
    assert oi == len(ops), (oi, len(ops), len(kernels))
    return rows


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:   # the table is still worth printing; say where the card line went
        return f"unknown ({e})"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("kind", choices=["sscd", "vit", "inception"])
    ap.add_argument("batch", type=int)
    ap.add_argument("--json", default=None, help="also write the rows here")
    args = ap.parse_args()
    import torch
    from torch.profiler import ProfilerActivity, profile
    from dcr_b200 import nets, synthetic
    from oracle import models as om
    assert torch.cuda.is_available(), "layer_profile measures on the GPU"
    kind, batch = args.kind, args.batch
    if kind == "sscd":
        net = nets.build_sscd_resnet50(om.make_sscd_state_dict(0), max_batch=batch,
                                       precision=os.environ.get("DCR_LP_PRECISION", "fast"))
        img = synthetic.images(32, seed=0)
    elif kind == "vit":
        net = nets.build_dino_vit(om.make_vit_state_dict(0), max_batch=batch)
        img = synthetic.images(32, seed=0)
    else:
        net = nets.build_fid_inception(om.make_inception_state_dict(0), max_batch=batch)
        img = torch.randint(0, 256, (32, 299, 299, 3), dtype=torch.uint8)
    img = img.cuda().repeat((batch + 31) // 32, 1, 1, 1)[:batch].contiguous()
    ops = describe(net.meta, batch)
    for _ in range(3):
        net(img)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(3):
            net(img)
        torch.cuda.synchronize()
    ev = [e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA and "dcr::" in e.name]
    ev.sort(key=lambda e: e.time_range.start)
    per = len(ev) // 3
    assert per * 3 == len(ev), len(ev)
    # per launch position: the median of the three forwards
    kernels = []
    for i in range(per):
        ts = sorted(ev[i + j * per].time_range.elapsed_us() for j in range(3))
        kernels.append((ev[i].name, ts[1]))
    rows = join(ops, kernels)
    tot = sum(r["us"] for r in rows)
    print(f"# {kind} batch {batch}: {card()}")
    print(f"{'op':12s} {'kernel':36s} {'M':>9s} {'N':>5s} {'K':>6s} {'us':>8s} {'TFLOP/s':>8s} {'GB/s':>7s} {'bound%':>7s} {'share%':>7s}")
    for r in rows:
        us = r["us"]
        bound_us = max(r["flops"] / PEAK_FLOPS, r["bytes"] / PEAK_BYTES) * 1e6
        r["bound_frac"] = bound_us / us if us else 0.0
        print(f"{r['op']:12s} {r['kernel'][:36]:36s} {r['M']:9d} {r['N']:5d} {r['K']:6d} {us:8.1f} "
              f"{r['flops'] / us / 1e6 if us else 0:8.1f} {r['bytes'] / us / 1e3 if us else 0:7.0f} "
              f"{100 * r['bound_frac']:7.1f} {100 * us / tot:7.1f}")
    print(f"total us {tot:.1f}  ({batch / tot * 1e6:.0f} img/s of kernel time)")
    fams = {}
    for r in rows:
        f = fams.setdefault(r["family"], [0, 0.0, 0.0, 0.0])
        f[0] += 1
        f[1] += r["us"]
        f[2] += r["flops"]
        f[3] += max(r["flops"] / PEAK_FLOPS, r["bytes"] / PEAK_BYTES) * 1e6
    print(f"{'family':28s} {'launches':>8s} {'us':>9s} {'share%':>7s} {'TFLOP/s':>8s} {'bound%':>7s}")
    for name, (n, us, fl, bu) in sorted(fams.items(), key=lambda kv: -kv[1][1]):
        print(f"{name:28s} {n:8d} {us:9.1f} {100 * us / tot:7.1f} {fl / us / 1e6:8.1f} {100 * bu / us:7.1f}")
    if args.json:
        os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
        with open(args.json, "w") as f:
            json.dump({"card": card(), "kind": kind, "batch": batch, "rows": rows}, f)


if __name__ == "__main__":
    main()
