"""Per-shape timing of the tensor-core convs at the C2 vocoder's shapes (LJSpeech iSTFTNet, B = 32, 512 frames).

    python tools/conv_tc_shapes.py [--reps 10] [--ablate] [--json OUT.json]

Every distinct Conv1d shape the vocoder's AdaIN resblocks and noise_res blocks run (256 ch at 10 240 frames,
128 ch at 61 441 frames; K = 3/7/11, dilation 1/3/5) plus conv_post, with seeded random weights, AdaIN coefficients and
Snake alphas, exactly as modules.AdaINResBlock1 calls ops.conv1d (dilation-1 shapes with the residual, like convs2).
Each shape is warmed up, then timed with CUDA events over --reps launches; the table gives ms per launch, algorithmic
TFLOP/s (2 * B * Cin * Cout * K * L) and the number of launches per C2 step.

--ablate repeats each shape under the kernel's timing switches (st2_debug_set_flags; their outputs are WRONG):
  4 = stagers skip the conversion, 16 = no weight copies, 32 = no raw activation copies.
The time a switch removes is the share of the role it disables that the other roles do not hide.
"""
import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch

B = 32
FRAMES = 512                     # C2: 128 tokens x 4 frames
ABLATIONS = {"no_convert": 4, "no_weights": 16, "no_raw": 32}


def c2_shapes():
    """(name, C_in, C_out, K, dil, L, residual, pre_act, launches per step)"""
    from styletts2_b200.lib import ACT_LRELU, ACT_SNAKE
    rows = []
    for ch, L, noise_k in ((256, 2 * FRAMES * 10, 7), (128, 2 * FRAMES * 60 + 1, 11)):
        blocks = [3, 7, 11, noise_k]          # the MRF resblocks, then noise_res
        for k in (3, 7, 11):
            nb = blocks.count(k)
            for d in (1, 3, 5):
                rows.append((f"rb c{ch} k{k} d{d}", ch, ch, k, d, L, d == 1, ACT_SNAKE, nb * (4 if d == 1 else 1)))
    rows.append(("conv_post", 128, 22, 7, 1, 2 * FRAMES * 60 + 1, False, ACT_LRELU, 1))
    return rows


def setup(ci, co, k, d, L, residual, pre_act, gen):
    from styletts2_b200 import ops
    from styletts2_b200.lib import ACT_SNAKE
    dev = "cuda"
    rn = dict(generator=gen, device=dev)
    w = (torch.rand(co, ci, k, **rn) * 2 - 1) / (ci * k) ** 0.5
    wt, wtc = ops.conv_weight_layout(w), ops.conv_tc_weight_layout(w)
    bias = torch.randn(co, **rn) * 0.1
    x = torch.randn(B, ci, L, **rn)
    res = torch.randn(B, co, L, **rn) if residual else None
    pre = (1 + 0.3 * torch.randn(B, ci, **rn), 0.3 * torch.randn(B, ci, **rn))
    alpha = 0.5 + torch.rand(1, ci, 1, **rn) if pre_act == ACT_SNAKE else None
    out = torch.empty(B, co, L, device=dev)
    pad = d * (k - 1) // 2
    kw = dict(K=k, dil=d, pad=pad, pre_act=pre_act, slope=0.01, alpha=alpha, res=res, out=out, want_stats=co != 22, wtc=wtc)
    if pre_act == ACT_SNAKE:
        kw["pre"] = pre

    def call():
        ops.conv1d(x, wt, bias, **kw)
    return call, wtc.mode


def time_ms(call, reps):
    for _ in range(2):
        call()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        call()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--ablate", action="store_true", help="also time each shape under the role-disabling switches")
    ap.add_argument("--json", default=None, help="write the rows to this JSON file")
    args = ap.parse_args()
    from styletts2_b200 import lib
    assert torch.cuda.is_available(), "needs a CUDA device"
    props = torch.cuda.get_device_properties(0)
    print(f"# {props.name}, B = {B}, {args.reps} timed launches per shape after 2 warm-up launches")
    ablations = ABLATIONS if args.ablate else {}
    print(f"{'shape':<18} {'kernel':<9} {'L':>6} {'ms':>8} {'TFLOP/s':>8} {'n/step':>6}" + "".join(f" {k:>11}" for k in ablations))
    gen = torch.Generator(device="cuda").manual_seed(0)
    rows, total = [], 0.0
    for name, ci, co, k, d, L, residual, act, n in c2_shapes():
        call, mode = setup(ci, co, k, d, L, residual, act, gen)
        ms = time_ms(call, args.reps)
        tf = 2.0 * B * ci * co * k * L / (ms / 1e3) / 1e12
        row = dict(shape=name, Cin=ci, Cout=co, K=k, dil=d, L=L, B=B, kernel="tct" if mode & lib.TC_TMAJOR else "tc",
                   ms=round(ms, 4), tflops=round(tf, 1), per_step=n)
        for key, flag in ablations.items():
            lib.call("st2_debug_set_flags", flag)
            try:
                row[key + "_ms"] = round(time_ms(call, args.reps), 4)
            finally:
                lib.call("st2_debug_set_flags", 0)
        total += ms * n
        rows.append(row)
        print(f"{name:<18} {row['kernel']:<9} {L:>6} {ms:>8.3f} {tf:>8.1f} {n:>6}" +
              "".join(f" {row[k + '_ms']:>11.3f}" for k in ablations), flush=True)
        torch.cuda.empty_cache()
    print(f"# sum of ms x launches per step over these shapes: {total:.1f} ms")
    if args.json:
        with open(args.json, "w") as f:
            json.dump(dict(device=props.name, B=B, reps=args.reps, rows=rows, ms_per_step=round(total, 2)), f, indent=1)


if __name__ == "__main__":
    main()
