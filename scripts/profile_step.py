#!/usr/bin/env python
"""Per-kernel profile of the headline workload's encoder (large-v2, one 3.84 s window: log-mel -> generate, beam 5)
under torch.profiler with CUDA activities.

Two profiled steps, each after its own warm-up:
  * enc_pdl=0: the encoder chain without programmatic dependent launch, so every kernel's duration is its own;
  * enc_pdl=1 (the production setting): dependents start early and wait inside, so their durations overlap and only
    the stage total (first kernel start to last kernel end) means something.

Writes under --out: launches_pdl{0,1}.csv (one row per encoder launch: role, kernel with template arguments, grid,
start, duration), summary.json, and prints a markdown summary per kernel family and GEMM role with achieved TFLOP/s
and L2->SM operand bytes per microsecond, both computed from the shapes below and the tile width / multicast flag read
from each GEMM's template arguments.

  python scripts/profile_step.py --out /tmp/encoder_profile
"""
import argparse
import csv
import json
import os
import re
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402
from willow_inference_server_b200 import _lib, weights as W  # noqa: E402

BM = 128  # GEMM tile rows (gemm_tc.cu)
T_PAD = 1536  # encoder rows per window
GEMM_ROLES = ("qkv", "out", "fc1", "fc2")


def gemm_shapes(d, n_dec_layers, windows=1):
    """(M, N, K) of every GEMM role of the encoder stage."""
    M = windows * T_PAD
    return {"conv2": (M, d, 3 * d), "qkv": (M, 3 * d, d), "out": (M, d, d), "fc1": (M, 4 * d, d), "fc2": (M, d, 4 * d),
            "cross_kv": (M, n_dec_layers * 2 * d, d)}


def operand_bytes(M, N, K, bn, mcast):
    """L2 -> SM operand bytes: every tile reads its 128 A rows and its BN W rows (half of them with 2-CTA multicast)."""
    tiles = (M // BM) * -(-N // bn)
    return tiles * (BM + (bn // 2 if mcast else bn)) * K * 2


def family(name):
    for key, fam in (("gemm_tc_kernel", "gemm"), ("enc_attn", "attention"), ("layernorm", "layernorm"),
                     ("conv1", "conv1")):
        if key in name:
            return fam
    return "other"


def gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=60).stdout.strip().splitlines()
        return q[0] if q else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def encoder_launches(trace_path, n_layers):
    """The kernels of one encoder stage, in launch order, tagged with their role."""
    with open(trace_path) as f:
        ev = json.load(f)["traceEvents"]
    ks = sorted((e for e in ev if e.get("cat") == "kernel"), key=lambda e: e["ts"])
    first = next(i for i, e in enumerate(ks) if "conv1" in e["name"])
    n = 2 + 7 * n_layers + 2  # conv1, conv2, per layer (ln, qkv, attn, out, ln, fc1, fc2), ln_post, cross-K/V
    chain = ks[first:first + n]
    roles = ["conv1", "conv2"]
    for _ in range(n_layers):
        roles += ["ln1", "qkv", "attn", "out", "ln2", "fc1", "fc2"]
    roles += ["ln_post", "cross_kv"]
    out = []
    for role, e in zip(roles, chain):
        fam = family(e["name"])
        want = "gemm" if role in ("conv2", "cross_kv") + GEMM_ROLES else None
        assert want is None or fam == "gemm", (role, e["name"])
        out.append(dict(role=role, family=fam, name=e["name"], grid=tuple(e.get("args", {}).get("grid", ())),
                        start_us=float(e["ts"]), dur_us=float(e["dur"])))
    assert len(out) == n, f"found {len(out)} of {n} encoder launches"
    return out


def summarise(launches, shapes, n_layers):
    t0 = launches[0]["start_us"]
    t1 = max(l["start_us"] + l["dur_us"] for l in launches)
    fams = {}
    for l in launches:
        fams[l["family"]] = fams.get(l["family"], 0.0) + l["dur_us"]
    roles = {}
    for role in ("conv2", *GEMM_ROLES, "cross_kv"):
        ls = [l for l in launches if l["role"] == role]
        m = re.search(r"gemm_tc_kernel<(\d+), *(true|false)>", ls[0]["name"])
        bn, mcast = int(m.group(1)), m.group(2) == "true"
        M, N, K = shapes[role]
        us = float(np.mean([l["dur_us"] for l in ls]))
        ob = operand_bytes(M, N, K, bn, mcast)
        roles[role] = dict(launches=len(ls), bn=bn, mcast=mcast, grid=ls[0]["grid"], mean_us=us,
                           total_us=us * len(ls), tflops=2.0 * M * N * K / us / 1e6, operand_MB=ob / 1e6,
                           operand_B_per_us=ob / us)
    for role in ("attn", "ln1", "ln2"):
        ls = [l for l in launches if l["role"] == role]
        roles[role] = dict(launches=len(ls), mean_us=float(np.mean([l["dur_us"] for l in ls])),
                           total_us=float(np.sum([l["dur_us"] for l in ls])))
    return dict(stage_us=t1 - t0, kernel_sum_us=sum(fams.values()), families=fams, roles=roles)


def print_summary(tag, s):
    print(f"\n### {tag}: stage {s['stage_us'] / 1e3:.3f} ms (first kernel start to last kernel end), "
          f"sum of kernel durations {s['kernel_sum_us'] / 1e3:.3f} ms")
    print("\n| family | ms | share of kernel sum |\n|---|---|---|")
    for f, us in sorted(s["families"].items(), key=lambda kv: -kv[1]):
        print(f"| {f} | {us / 1e3:.3f} | {100 * us / s['kernel_sum_us']:.1f} % |")
    print("\n| role | launches | plan (BN, mcast) | grid | mean µs | total ms | TFLOP/s | operand MB | operand B/µs |")
    print("|---|---|---|---|---|---|---|---|---|")
    for role, r in s["roles"].items():
        if "bn" in r:
            print(f"| {role} | {r['launches']} | {r['bn']}, {int(r['mcast'])} | {r['grid'][0] if r['grid'] else '?'} | "
                  f"{r['mean_us']:.1f} | {r['total_us'] / 1e3:.3f} | {r['tflops']:.0f} | {r['operand_MB']:.0f} | "
                  f"{r['operand_B_per_us']:.3g} |")
        else:
            print(f"| {role} | {r['launches']} | | | {r['mean_us']:.1f} | {r['total_us'] / 1e3:.3f} | | | |")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True, help="output directory (created)")
    ap.add_argument("--model", default="large-v2")
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()

    import torch
    from torch.profiler import ProfilerActivity, profile

    os.makedirs(args.out, exist_ok=True)
    info = gpu_info()
    print("GPU (name, power limit, max SM clock):", info)
    dims = W.WhisperDims.for_size(args.model)
    shapes = gemm_shapes(dims.d_model, dims.n_dec_layers)
    host, _ = bench.make_blob_host(dims)
    h = _lib.Handle.from_host(host.numpy(), 0)
    pcm = torch.from_numpy(bench.synth_utterance(bench.AUDIO_SAMPLES, 1234)).cuda()
    off, ns = np.zeros(1, np.int64), np.array([bench.AUDIO_SAMPLES], np.int32)
    prompts = np.array([bench.PROMPT], np.int32)

    def step():
        h.logmel(pcm.data_ptr(), off, ns, to_host=False, keep=True, pcm_on_device=True, pcm_dtype=_lib.PCM_F32, B=1)
        h.generate(None, prompts, bench.BEAM, 1.0, 1.0, bench.MAX_LENGTH, [dims.eot], B=1)

    result = {"gpu": info, "model": args.model}
    for pdl in (0, 1):
        h.set_option("enc_pdl", pdl)
        for _ in range(args.warmup):
            step()
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            step()
            torch.cuda.synchronize()
        trace = os.path.join(args.out, f"trace_pdl{pdl}.json")
        prof.export_chrome_trace(trace)
        launches = encoder_launches(trace, dims.n_enc_layers)
        os.remove(trace)  # large; the table below keeps what matters
        with open(os.path.join(args.out, f"launches_pdl{pdl}.csv"), "w", newline="") as f:
            w = csv.writer(f)
            w.writerow(["role", "kernel", "grid", "start_us", "dur_us"])
            for l in launches:
                w.writerow([l["role"], l["name"], "x".join(map(str, l["grid"])), f"{l['start_us'] - launches[0]['start_us']:.2f}",
                            f"{l['dur_us']:.2f}"])
        s = summarise(launches, shapes, dims.n_enc_layers)
        s["timing_ms"] = h.timing()
        result[f"pdl{pdl}"] = s
        print_summary(f"enc_pdl={pdl}", s)
    with open(os.path.join(args.out, "summary.json"), "w") as f:
        json.dump(result, f, indent=1, default=str)


if __name__ == "__main__":
    main()
