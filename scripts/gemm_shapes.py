"""Per-shape time of the tensor-core GEMM / convolution kernel (tc_gemm_kernel) over one dense pass of the benchmark.

Builds the benchmark's system (bench.build_system: 512^2 renders, 8 views, fp16 by default) and runs the dense section
once eagerly -- VAE encode, ControlNet + UNet over the 3-branch batch with the fused CSD epilogue, VAE backward -- with
dense_ops.gemm / conv2d / conv2d_csd wrapped so that every call records its shape, epilogue and tile plan
(dm_gemm_plan: tile width BN and split-K).  Identical calls are merged; each distinct call is then replayed alone, with
its own tensors, as a CUDA graph of --iters launches (the benchmark replays the dense section from graphs too), timed
with CUDA events after a warm-up.

One row per shape: calls per step, time per call and per step, share of the summed GEMM time, achieved TFLOP/s and GB/s
from algorithmic FLOPs and bytes (operands read once, output and residual once; no split-K workspace, no L2 effects),
the roof that bounds the shape and the fraction of it reached.  The roofs are the H100 SXM data sheet's dense fp16/bf16
rate and HBM3 bandwidth; the card's name and power limit are printed with the table.

    python scripts/gemm_shapes.py [--iters 20] [--dtype f16|bf16] [--json OUT.json]
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

PEAK_TFLOPS = 989.0     # H100 SXM data sheet, dense fp16 / bf16 tensor core
PEAK_GBS = 3350.0       # H100 SXM data sheet, HBM3


def card():
    name = torch.cuda.get_device_name()
    try:
        q = subprocess.run(["nvidia-smi", "-i", str(torch.cuda.current_device()),
                            "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as ex:  # noqa: BLE001 -- the table stands without it, but says so
        q = f"nvidia-smi unavailable ({ex})"
    return f"{name}, power limit / max SM clock: {q}"


def plan(M, N, K, act, bn_hint):
    from dreammat_b200._cabi import check, lib
    k, bn, sp = C.c_int(), C.c_int(), C.c_int()
    check(lib().dm_gemm_plan(M, N, K, act, bn_hint, C.byref(k), C.byref(bn), C.byref(sp)), "dm_gemm_plan")
    return bn.value, sp.value


def describe_gemm(a, b, kw):
    from dreammat_b200 import dense_ops as D
    batch = a.shape[0] if a.dim() == 3 else 1
    M, K, N = a.shape[-2], a.shape[-1], b.shape[-2]
    act = kw.get("act")
    out = kw.get("out")
    out_f32 = kw.get("out_f32", False) or (out is not None and out.dtype == torch.float32)
    n_out = N // 2 if act == "geglu" else N
    es = a.element_size()
    b_batched = b.dim() == 3
    byts = (batch * M * K + (batch if b_batched else 1) * N * K) * es + batch * M * n_out * (4 if out_f32 else es)
    if kw.get("residual") is not None:
        byts += batch * M * N * es
    if kw.get("bias") is not None:
        byts += N * es
    if kw.get("rowvec") is not None:
        byts += kw["rowvec"].numel() * es
    # a shared B folds the batch into M; a batched B keeps it on grid.z (the plan sees M * batch either way)
    bn, split = plan(M * batch, N, K, D.ACT[act], kw.get("bn", 0))
    shape = (f"{batch}x " if batch > 1 else "") + f"{M}x{N}x{K}" + (" Bb" if b_batched else "")
    return dict(kind="gemm", shape=shape, M=M * batch, N=N, K=K, batch=batch, flops=2.0 * batch * M * N * K, bytes=byts,
                bn=bn, split=split, epilogue=_ep_text(kw, out_f32))


def describe_conv(x, w, ksize, kw):
    from dreammat_b200 import dense_ops as D
    n, H, W, Cin = x.shape
    Cout = w.shape[0]
    stride = kw.get("stride", 1)
    pad = kw.get("pad", (1, 1))
    if kw.get("out_hw") is not None:
        Ho, Wo = kw["out_hw"]
    else:
        Ho, Wo = (H + 2 * pad[0] - ksize) // stride + 1, (W + 2 * pad[1] - ksize) // stride + 1
    out = kw.get("out")
    out_f32 = kw.get("out_f32", False) or (out is not None and out.dtype == torch.float32)
    es = x.element_size()
    M, K = n * Ho * Wo, ksize * ksize * Cin
    byts = (x.numel() + w.numel()) * es + M * Cout * (4 if out_f32 else es)
    if kw.get("residual") is not None:
        byts += M * Cout * es
    if kw.get("rowvec") is not None:
        byts += kw["rowvec"].numel() * es
    bn, split = plan(M, Cout, K, D.ACT[kw.get("act")], kw.get("bn", 0))
    shape = f"conv{ksize}x{ksize}s{stride} {n}x{H}x{W} {Cin}->{Cout}"
    return dict(kind="conv", shape=shape, M=M, N=Cout, K=K, batch=1, flops=2.0 * M * Cout * K, bytes=byts, bn=bn,
                split=split, epilogue=_ep_text(kw, out_f32))


def describe_csd(x, w, noise, eps_out):
    n3, h, ww, Cin = x.shape
    B = n3 // 3
    M, K = n3 * h * ww, 9 * Cin
    # input, weights, noise read; grad and dlatents written (fp32, NCHW); eps written when kept for debugging
    byts = (x.numel() + w.numel()) * x.element_size() + 3 * noise.numel() * 4 + (eps_out.numel() * 4 if eps_out is not None else 0)
    return dict(kind="csd", shape=f"conv3x3s1+csd {n3}x{h}x{ww} {Cin}->4", M=M, N=4, K=K, batch=1,
                flops=2.0 * M * 4 * K, bytes=byts, bn=64, split=1, epilogue="csd")


def _ep_text(kw, out_f32):
    parts = [k for k in ("bias", "rowvec", "residual") if kw.get(k) is not None]
    if kw.get("act"):
        parts.append(kw["act"])
    if kw.get("alpha", 1.0) != 1.0 or kw.get("out_scale", 1.0) != 1.0:
        parts.append("scale")
    if out_f32:
        parts.append("f32")
    out = kw.get("out")
    if out is not None and out.stride(-2) != out.shape[-1]:
        parts.append("ldc")
    return "+".join(parts) or "-"


def _key(args, kw):
    """everything that decides the kernel's work: shapes, strides, dtypes, which epilogue terms are present"""
    def k(v):
        if torch.is_tensor(v):
            return ("T", tuple(v.shape), tuple(v.stride()), str(v.dtype))
        if isinstance(v, (list, tuple)):
            return tuple(k(x) for x in v)
        return v
    return tuple(k(a) for a in args) + tuple(sorted((n, k(v)) for n, v in kw.items()))


class Recorder:
    def __init__(self):
        self.rows = {}

    def wrap(self, D):
        orig = {"gemm": D.gemm, "conv2d": D.conv2d, "conv2d_csd": D.conv2d_csd}

        def rec(name, describe):
            fn = orig[name]

            def wrapped(*args, **kw):
                key = (name, _key(args, kw))
                r = self.rows.get(key)
                if r is None:
                    r = self.rows[key] = dict(describe(*args, **kw), calls=0, replay=(fn, args, kw))
                r["calls"] += 1
                return fn(*args, **kw)
            return wrapped

        D.gemm = rec("gemm", lambda a, b, **kw: describe_gemm(a, b, kw))
        D.conv2d = rec("conv2d", lambda x, w, ksize, **kw: describe_conv(x, w, ksize, kw))
        D.conv2d_csd = rec("conv2d_csd", lambda x, w, bias, noise, w1mac, coef, **kw: describe_csd(x, w, noise, kw.get("eps_out")))
        return orig


def dense_pass(sysm, cams, views, dev):
    """the eager dense section of DreamMat.training_step_fused: VAE encode with grad, ControlNet + UNet x3 (CSD fused),
    VAE backward"""
    from dreammat_b200.guidance import _SDSLoss
    from dreammat_b200.scene import FixViewMaps
    guid = sysm.guidance
    guid.update_step(0, 0)
    maps = FixViewMaps.synthetic(cams.cfg.fix_view_num, cams.cfg.fix_env_num, 512, 512, device=dev, seed=7)
    guid.maps = maps
    view_id, env_id = cams.collate(torch.Generator().manual_seed(1234), views)
    c = cams.cameras(view_id)
    ctx3 = sysm.prompt_utils.get_text_embeddings(c["elevation"].to(dev), c["azimuth"].to(dev), c["camera_distances"].to(dev),
                                                 guid.cfg.view_dependent_prompting, return_null_text_embeddings=True)
    cond = maps.condition_map(view_id, env_id)
    rgb = torch.rand(views, 512, 512, 3, device=dev, generator=torch.Generator(device=dev).manual_seed(5)).requires_grad_(True)
    lat = guid.encode_images(rgb)
    grad, dlat, sums = guid.compute_grad_sds(lat, cond, ctx3)
    loss = _SDSLoss.apply(lat, dlat, sums[0] / views)
    loss.backward()
    torch.cuda.synchronize()


def time_call(fn, args, kw, iters, warmup=3):
    for _ in range(warmup):
        fn(*args, **kw)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for _ in range(iters):
            fn(*args, **kw)
    g.replay()                       # first replay uploads the graph
    torch.cuda.synchronize()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    g.replay()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e) * 1e3 / iters      # us per call


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--views", type=int, default=8)
    ap.add_argument("--dtype", default="f16", choices=["f16", "bf16"])
    ap.add_argument("--json", help="also write the rows to this file")
    args = ap.parse_args()
    assert args.iters >= 20, "at least 20 launches per shape"
    if not torch.cuda.is_available():
        sys.exit("gemm_shapes.py times kernels on the GPU; no CUDA device found")
    dev = "cuda:0"
    torch.cuda.set_device(0)
    torch.manual_seed(0)
    import bench
    from dreammat_b200 import dense_ops as D
    dtype = torch.bfloat16 if args.dtype == "bf16" else torch.float16
    sysm, cams = bench.build_system(dev, 512, 20000, (256, 512), 0, dtype)
    rec = Recorder()
    orig = rec.wrap(D)
    try:
        dense_pass(sysm, cams, args.views, dev)
    finally:
        D.gemm, D.conv2d, D.conv2d_csd = orig["gemm"], orig["conv2d"], orig["conv2d_csd"]
    rows = list(rec.rows.values())
    for r in rows:
        fn, a, kw = r.pop("replay")
        r["us"] = time_call(fn, a, kw, args.iters)
        r["ms_step"] = r["us"] * r["calls"] / 1e3
        r["tflops"] = r["flops"] / (r["us"] * 1e-6) / 1e12
        r["gbs"] = r["bytes"] / (r["us"] * 1e-6) / 1e9
        t_mma, t_hbm = r["flops"] / (PEAK_TFLOPS * 1e12), r["bytes"] / (PEAK_GBS * 1e9)
        r["bound"] = "mma" if t_mma >= t_hbm else "hbm"
        r["roof_frac"] = max(t_mma, t_hbm) / (r["us"] * 1e-6)
    total = sum(r["ms_step"] for r in rows)
    for r in rows:
        r["share"] = r["ms_step"] / total
    rows.sort(key=lambda r: -r["ms_step"])
    info = card()
    print(f"# {info}")
    print(f"# {len(rows)} shapes, {sum(r['calls'] for r in rows)} calls per step, {total:.2f} ms of GEMM time per step "
          f"({args.dtype}, {args.views} views at 512^2; CUDA-graph replay of {args.iters} launches per shape)")
    hdr = f"{'shape':40s} {'epilogue':24s} {'BN':>3s} {'spl':>3s} {'calls':>5s} {'us/call':>9s} {'ms/step':>8s} " \
          f"{'share':>6s} {'TFLOP/s':>8s} {'GB/s':>7s} {'bound':>5s} {'roof':>6s}"
    print(hdr)
    for r in rows:
        print(f"{r['shape']:40s} {r['epilogue']:24s} {r['bn']:3d} {r['split']:3d} {r['calls']:5d} {r['us']:9.1f} "
              f"{r['ms_step']:8.3f} {100 * r['share']:5.1f}% {r['tflops']:8.1f} {r['gbs']:7.0f} {r['bound']:>5s} "
              f"{100 * r['roof_frac']:5.1f}%")
    if args.json:
        with open(args.json, "w") as f:
            json.dump({"card": info, "dtype": args.dtype, "views": args.views, "iters": args.iters,
                       "total_ms_step": total, "rows": rows}, f, indent=1)


if __name__ == "__main__":
    main()
