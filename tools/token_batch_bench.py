"""Text-side time of a queue of utterances with different token counts, two ways:
  (a) buckets of exactly equal token count (parallel.plan_equal_length_batches: no token padding inside a batch), one
      synthesize call per bucket;
  (b) the whole queue as one batch with the style sampler on packed token rows (synthesize(..., token_packing=True)).
The text side is the span from a call's start to its `duration` stage mark (text encoder, bert_encoder, sampler,
duration predictor; `bert_dur` is an input, as in bench.py), timed with CUDA events after a warm-up of every shape; (a)
sums it over its buckets.  Both ways get the same per-utterance step noises, and the largest s_pred difference between
them is reported (every utterance gets its single-utterance style either way).  Runs (a) and (b) alternately --repeats
times and prints one JSON object with every run, the card, its power limit and the SM clocks sampled during the runs.

Usage: python tools/token_batch_bench.py [--model ljspeech] [--utterances 32] [--repeats 3] [--out FILE]"""
import argparse
import json
import os
import random
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle"))


def gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:                       # noqa: BLE001
        q = f"nvidia-smi unavailable ({e})"
    return {"nvidia_smi": q, "torch_name": torch.cuda.get_device_name(0)}


def queue(n, seed, multispeaker, lo=16, hi=256):
    r = random.Random(seed)
    lengths = [r.randint(lo, hi) for _ in range(n)]
    g = torch.Generator().manual_seed(seed)
    toks = [[0] + torch.randint(1, 178, (m - 1,), generator=g).tolist() for m in lengths]
    bert = [torch.randn(m, 768, generator=g) * 0.5 for m in lengths]
    noise = torch.randn(n, 1, 256, generator=g)
    ref_s = torch.randn(n, 256, generator=g) * 0.5 if multispeaker else None
    return lengths, toks, bert, noise, ref_s


def batch_inputs(idx, toks, bert, noise, ref_s, steps, dev):
    lens = [len(toks[i]) for i in idx]
    B, N = len(idx), max(lens)
    tk = torch.zeros(B, N, dtype=torch.long)
    bd = torch.zeros(B, N, 768)
    for j, i in enumerate(idx):
        tk[j, :lens[j]] = torch.tensor(toks[i])
        bd[j, :lens[j]] = bert[i]
    ii = torch.tensor(idx)
    args = (tk.to(dev), torch.tensor(lens).to(dev), bd.to(dev), noise[ii].to(dev))
    return args, None if ref_s is None else ref_s[ii].to(dev), [s[ii].to(dev) for s in steps]


def text_side_ms(syn, args, ref_s, steps, K, packing):
    """one synthesize call (durations pinned to 1 frame per token: the tail stays short) -> (start..duration ms, s_pred)"""
    marks = []
    out = syn.synthesize(*args, diffusion_steps=K, ref_s=ref_s, rng=dict(step_noises=steps), pin_frames_per_token=1,
                         stage_marks=marks, return_all=True, token_packing=packing)
    torch.cuda.synchronize()
    ev = dict(marks)
    return ev["start"].elapsed_time(ev["duration"]), out["s_pred"]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--model", default="ljspeech", choices=["ljspeech", "libritts"])
    ap.add_argument("--utterances", type=int, default=32)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--seed", type=int, default=1)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "token_batch_bench needs a GPU"
    import cases
    from bench import ClockSampler
    from styletts2_b200.inference import Synthesizer
    from styletts2_b200.models import build_model, load_keyed_weights, recursive_munch
    from styletts2_b200.parallel import plan_equal_length_batches
    dev = "cuda:0"
    mcfg = cases.MODEL_CFGS[a.model]
    m = build_model(recursive_munch(mcfg))
    for k in m:
        m[k].to(dev).eval()
    load_keyed_weights(m)
    syn = Synthesizer(m, mcfg, dev)
    n, K = a.utterances, a.steps
    lengths, toks, bert, noise, ref_s = queue(n, a.seed, bool(mcfg["multispeaker"]))
    g = torch.Generator().manual_seed(a.seed + 1)
    steps = [torch.randn(n, 1, 256, generator=g) for _ in range(K - 1)]
    buckets = plan_equal_length_batches(lengths, 1, n)[0]
    ins_a = [(idx, batch_inputs(idx, toks, bert, noise, ref_s, steps, dev)) for idx in buckets]
    all_idx = list(range(n))
    ins_b = batch_inputs(all_idx, toks, bert, noise, ref_s, steps, dev)

    def run_a():
        total, s = 0.0, torch.empty(n, 256, device=dev)
        for idx, (args, rs, st) in ins_a:
            ms, sp = text_side_ms(syn, args, rs, st, K, False)
            total += ms
            s[torch.tensor(idx, device=dev)] = sp
        return total, s

    def run_b():
        args, rs, st = ins_b
        return text_side_ms(syn, args, rs, st, K, True)

    with torch.no_grad():
        for _ in range(2):                       # warm-up: every bucket shape and the packed batch
            run_a()
            run_b()
        clocks = ClockSampler(0)
        clocks.start()
        runs = []
        for _ in range(a.repeats):
            ta, sa = run_a()
            tb, sb = run_b()
            runs.append({"a_buckets_ms": ta, "b_packed_ms": tb, "a_over_b": ta / tb,
                         "s_pred_maxabs_a_vs_b": float((sa - sb).abs().max())})
        clk = clocks.stop()
    res = {"model": a.model, "utterances": n, "diffusion_steps": K, "token_counts": lengths, "distinct_token_counts": len(buckets),
           "tokens": sum(lengths), "runs": runs, "gpu": gpu_info(), "clocks": clk}
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
