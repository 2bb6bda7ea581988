"""Per-tile cost of the tensor-core conv kernels, fitted against the number of taps, from a per-shape table.

    python tools/conv_tc_shapes.py --json shapes.json      # on the GPU
    python tools/conv_tc_fit.py shapes.json [--sms 132] [--ghz 1.48]

A persistent CTA per SM loops over 128-frame tiles, and each tile runs one MMA step per (tap, 16-channel block).  For the
shapes that differ only in K (same kernel, channels and dilation) this fits

    ms per launch / tiles per SM  =  slope * K * ceil(Cin / 16)  +  fixed

by least squares.  `slope` is the time of one (tap, block) step, given in cycles at --ghz; `fixed` is the part of a tile
that does not depend on K (epilogue, hand-offs, pipeline start).  The last columns weight `fixed` by tiles and launches per
step: the share of the step that a smaller per-tile cost would give back.
"""
import argparse
import json
import math
from collections import defaultdict

import numpy as np

TN, CB, TM = 128, 16, 128   # frames per tile, input channels per block, output channels per channel-major tile


def tiles(row):
    n = row["B"] * math.ceil(row["L"] / TN)
    return n if row["kernel"] == "tct" else n * math.ceil(row["Cout"] / TM)


def fit(rows, sms, ghz):
    groups = defaultdict(list)
    for r in rows:
        groups[(r["kernel"], r["Cin"], r["Cout"], r["dil"], r["shape"].split()[0])].append(r)
    out = []
    for (kern, ci, co, dil, _), rs in sorted(groups.items()):
        if len({r["K"] for r in rs}) < 2:
            continue
        rs = sorted(rs, key=lambda r: r["K"])
        per_sm = [tiles(r) / sms for r in rs]
        us = np.array([r["ms"] * 1e3 / t for r, t in zip(rs, per_sm)])
        steps = np.array([r["K"] * math.ceil(ci / CB) for r in rs], dtype=float)
        slope, fixed = np.polyfit(steps, us, 1)
        fixed_ms = sum(fixed * t / 1e3 * r["per_step"] for r, t in zip(rs, per_sm))
        total_ms = sum(r["ms"] * r["per_step"] for r in rs)
        out.append(dict(kernel=kern, Cin=ci, Cout=co, dil=dil, K=[r["K"] for r in rs], us_per_tile=[round(float(u), 1) for u in us],
                        slope_cycles=slope * ghz * 1e3, fixed_us=fixed, fixed_ms_per_step=fixed_ms, ms_per_step=total_ms))
    return out


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("json", help="output of tools/conv_tc_shapes.py --json")
    ap.add_argument("--sms", type=int, default=132, help="persistent CTAs (SMs of the GPU the table was measured on)")
    ap.add_argument("--ghz", type=float, default=1.48, help="SM clock used to express the slope in cycles")
    args = ap.parse_args()
    with open(args.json) as f:
        d = json.load(f)
    print(f"# {d.get('device', '?')}, B = {d.get('B', '?')}, {args.sms} SMs, cycles at {args.ghz} GHz")
    print(f"{'kernel':<6} {'Cin':>4} {'Cout':>4} {'dil':>3}  {'us per tile at K':<24} {'slope (cyc/step)':>16} {'fixed us/tile':>13}"
          f" {'fixed ms/step':>13} {'of ms/step':>10}")
    for r in fit(d["rows"], args.sms, args.ghz):
        ks = " / ".join(f"{u:.1f}" for u in r["us_per_tile"]) + " (" + "/".join(map(str, r["K"])) + ")"
        print(f"{r['kernel']:<6} {r['Cin']:>4} {r['Cout']:>4} {r['dil']:>3}  {ks:<24} {r['slope_cycles']:>16.0f} {r['fixed_us']:>13.1f}"
              f" {r['fixed_ms_per_step']:>13.1f} {r['ms_per_step']:>10.1f}")


if __name__ == "__main__":
    main()
