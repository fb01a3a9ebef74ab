"""Time per wavefront-loop iteration of each kernel next to its traffic floor, on C1 (bench.py's scene, seed and tiles).

The floor of a kernel is the bytes it has to move per unit of work (bench.STREAM_BYTES, plus PREP_BYTES per shadow query for
k_shadow_prep and SORT_BYTES per survivor for the coherence sort) over the device-to-device copy bandwidth measured in the same
run.  Times are the library's CUDA-event profile (tgb200_set_profiling), summed over both wavefronts and divided by the
iterations of both, so a kernel's time includes whatever the other wavefront's kernels take from it.  The traversal kernels
have no traffic floor here (they are issue bound, DESIGN.md section 5); their times are printed for scale.

    python tools/loop_floor.py [--steps 4] [--warmup 1] [--json out.json]
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402

# k_shadow_prep: queue entry (4) + shading point and direction (32) read, light index (16-byte record, 4 used) ~ 8, queue
# entry + cut mask or analytic hit written (~16); the coherence sort: key read (4), cursor update (4), order entry written (4)
PREP_BYTES, SORT_BYTES = 60, 12


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        name, power, clock = [s.strip() for s in out[0].split(",")]
        return {"gpu": name, "power_limit": power, "sm_max_clock": clock}
    except Exception as e:                                      # the numbers still print without the card's settings
        return {"gpu": None, "error": str(e)[:120]}


def copy_bandwidth(torch, nbytes=1 << 30, reps=10):
    """Best device-to-device copy rate over `reps` copies of `nbytes`, bytes read + written per second."""
    a = torch.empty(nbytes, dtype=torch.uint8, device="cuda"); b = torch.empty_like(a)
    b.copy_(a); torch.cuda.synchronize()
    best = None
    for _ in range(reps):
        e0 = torch.cuda.Event(enable_timing=True); e1 = torch.cuda.Event(enable_timing=True)
        e0.record(); b.copy_(a); e1.record(); torch.cuda.synchronize()
        t = e0.elapsed_time(e1)/1e3
        best = t if best is None else min(best, t)
    return 2*nbytes/best


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=4)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--spp-per-step", type=int, default=64)
    ap.add_argument("--json", default=None, help="also write the table to this file")
    args = ap.parse_args()

    import torch
    from tungsten_b200 import integrator, lib, scene
    if not torch.cuda.is_available():
        raise SystemExit("loop_floor.py needs a CUDA device")
    W, H = bench.CONFIGS["c1"]["res"]
    bench.W, bench.H = W, H
    seed = 0xBA5EBA11
    ctx = lib.Context(scene.load_scene(bench.make_scene(1024, "c1")), device=0)
    tiles = integrator.dice_tiles(W, H, seed)
    spp = args.spp_per_step
    for i in range(args.warmup):
        ctx.render_resident(spp, seed=seed, spp_begin=i*spp, tiles=tiles)
    ctx.clear(); ctx.reset_stats(); ctx.set_profiling(True)
    for i in range(args.steps):
        ctx.render_resident(spp, seed=seed, spp_begin=i*spp, tiles=tiles)
    torch.cuda.synchronize()
    st = ctx.stats()
    ctx.close()
    bw = copy_bandwidth(torch)

    it = max(int(st.iterations), 1)
    survivors = float(st.path_rays) - float(st.samples)
    rows = [  # kernel, ms, units, bytes per unit
        ("k_regen", st.regen_ms, float(st.samples), bench.STREAM_BYTES["k_regen"]["bytes_per_unit"]),
        ("k_shade", st.shade_ms, float(st.path_rays), bench.STREAM_BYTES["k_shade"]["bytes_per_unit"]),
        ("k_shadow_prep", st.prep_ms, float(st.shadow_rays), PREP_BYTES),
        ("k_accum", st.accum_ms, float(st.path_rays), bench.STREAM_BYTES["k_accum"]["bytes_per_unit"]),
        ("k_iter_end + k_bin_scatter", st.sort_ms, survivors, SORT_BYTES),
        ("k_trace", st.trace_ms, float(st.path_rays_traversed), None),
        ("k_shadow_bvh", st.shadow_ms, float(st.shadow_rays_traversed), None),
    ]
    out = {"card": card(), "copy_gbs": bw/1e9, "steps": args.steps, "spp_per_step": spp, "iterations": it,
           "total_ms": st.total_ms, "samples": int(st.samples), "kernels": []}
    print("%s, power limit %s, max SM clock %s; copy bandwidth %.0f GB/s; %d steps x %d spp, %d iterations (both wavefronts)"
          % (out["card"].get("gpu"), out["card"].get("power_limit"), out["card"].get("sm_max_clock"), bw/1e9, args.steps, spp, it))
    print("%-28s %10s %12s %12s %10s %8s" % ("kernel", "ms", "us/iter", "floor us/it", "GB/s", "x floor"))
    for name, ms, units, bpu in rows:
        us = 1e3*ms/it
        row = {"kernel": name, "ms": ms, "us_per_iter": us, "units": units, "bytes_per_unit": bpu}
        if bpu is not None:
            floor_us = 1e6*units*bpu/bw/it
            row.update(floor_us_per_iter=floor_us, gbs=units*bpu/1e9/(ms/1e3) if ms > 0 else 0.0)
            print("%-28s %10.1f %12.1f %12.1f %10.0f %8.2f" % (name, ms, us, floor_us, row["gbs"], us/floor_us if floor_us > 0 else 0.0))
        else:
            print("%-28s %10.1f %12.1f %12s %10s %8s" % (name, ms, us, "-", "-", "-"))
        out["kernels"].append(row)
    if args.json:
        with open(args.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
