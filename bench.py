"""Benchmark of the StyleTTS 2 text->waveform hot path on H100 (one JSON result line per run).

    python bench.py --gpus N --steps K --warmup W            # this repo's CUDA path (default workload C2 per GPU)
    python bench.py --impl reference --steps K --warmup W    # the reference algorithm on host cores (oracle port)
    python bench.py --workload C3 --global-batch 64 --gather # BASELINE configs[2]: B=64 sharded by utterance over the ranks
    python bench.py --workload C5 --diffusion-steps 50       # BASELINE configs[4]: diffusion-step sweep point

A "step" = one pass of the whole path (text encoder -> style diffusion sampler -> duration/prosody predictor ->
AdaIN decoder -> vocoder) over one batch of synthetic utterances.  Default workload = BASELINE.json configs[1]:
LJSpeech config, iSTFTNet decoder, batch 32 x 128 tokens x 512 frames (4 frames/token pinned after the duration
kernel has run, SURVEY section 8d), diffusion_steps=5.  Weights: key-seeded random init of that architecture
(no checkpoints offline).  With N>1 and no --global-batch every rank runs the same per-GPU batch (weak scaling,
utterance sharding, no data-path collective); with --global-batch the batch is split by parallel.shard_range (strong).
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import torch  # noqa: E402

WORKLOADS = {
    # name: model cfg, per-GPU batch (or global batch with --global-batch), tokens, frames/token, diffusion steps
    "C2": dict(model="ljspeech", B=32, N=128, fpt=4, steps=5, desc="LJSpeech iSTFTNet B32 N128 T512 K5"),
    "C3": dict(model="libritts", B=8, N=128, fpt=4, steps=10, desc="LibriTTS HiFi-GAN B8/GPU (global 64 on 8 GPUs) N128 T512 K10"),
    "C4": dict(model="ljspeech", B=16, N=500, fpt=4, steps=5, desc="LJSpeech iSTFTNet B16 N500 T2000 K5"),
    "C5": dict(model="ljspeech", B=8, N=128, fpt=4, steps=5, desc="diffusion-step sweep point, B8/GPU (global 64 on 8 GPUs) N128 T512"),
    "tiny": dict(model="ljspeech", B=2, N=16, fpt=4, steps=3, desc="plumbing check"),
}
# SURVEY section 8(d): algorithmic bytes / FLOPs of the decoder+vocoder path per frame-utterance (fp32, conv
# boundaries, norm/activation/residual fused) + weights once per launch chain.
VOCODER_BYTES_PER_FRAME = {"ljspeech": 4.445e6, "libritts": 11.74e6}
VOCODER_WEIGHT_BYTES = {"ljspeech": 223e6, "libritts": 224e6}
VOCODER_FLOPS_PER_FRAME = {"ljspeech": 1.317e9, "libritts": 1.767e9}


def denoiser_flops(N, K, cfg_scale=1.0):
    """SURVEY 8(d): 37.8e6*N + 6144*N^2 per (utterance, eval); evals = 2(K-1) (x2 with classifier-free guidance)."""
    return (37.8e6 * N + 6144.0 * N * N) * 2 * (K - 1) * (2 if cfg_scale != 1.0 else 1)


def measured_peaks():
    """(hbm GB/s, sustained bf16 TFLOP/s, burst bf16 TFLOP/s, source): kernels timed inside a long step -> sustained."""
    p = os.path.join(ROOT, "MEASURED_PEAKS.json")
    if os.path.exists(p):
        d = json.load(open(p))
        return (float(d["hbm_gbs"]), float(d.get("bf16_tflops_sustained", d["bf16_tflops"])), float(d["bf16_tflops"]),
                "measured (MEASURED_PEAKS.json: copy GB/s, sustained cuBLAS bf16)")
    return 3350.0, 989.0, 989.0, "H100 SXM data sheet (dense bf16, HBM3), not a measurement"


def ncu_traffic():
    """DRAM bytes per launch of the dominant kernel from the committed ncu --set full capture (profiles/), or None."""
    p = os.path.join(ROOT, "profiles", "r02_ncu_traffic.json")
    if os.path.exists(p):
        return json.load(open(p))
    return None


class ClockSampler:
    """nvidia-smi clocks/throttle reasons sampled DURING the timed region."""
    Q = "clocks.sm,clocks.max.sm,clocks_event_reasons.hw_slowdown,clocks_event_reasons.hw_thermal_slowdown," \
        "clocks_event_reasons.sw_thermal_slowdown,clocks_event_reasons.sw_power_cap"

    def __init__(self, index):
        self.index, self.proc, self.path = index, None, None

    def start(self):
        try:
            f = tempfile.NamedTemporaryFile("w", suffix=".csv", delete=False)
            self.path = f.name
            self.proc = subprocess.Popen(["nvidia-smi", "-i", str(self.index), f"--query-gpu={self.Q}", "--format=csv,noheader,nounits",
                                          "-lms", "100"], stdout=f, stderr=subprocess.DEVNULL)
        except Exception:
            self.proc = None

    def stop(self):
        if self.proc is None:
            return {"sm_mhz": None, "sm_max_mhz": None, "reasons": ["nvidia-smi unavailable"]}
        self.proc.terminate()
        try:
            self.proc.wait(timeout=5)
        except Exception:
            self.proc.kill()
        sm, mx, reasons = [], [], set()
        for line in open(self.path):
            parts = [x.strip() for x in line.split(",")]
            if len(parts) < 6:
                continue
            try:
                sm.append(float(parts[0])); mx.append(float(parts[1]))
            except ValueError:
                continue
            for name, v in zip(["hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown", "sw_power_cap"], parts[2:6]):
                if v.lower().startswith("active"):
                    reasons.add(name)
        os.unlink(self.path)
        sm.sort()
        return {"sm_mhz": sm[len(sm) // 2] if sm else None, "sm_max_mhz": max(mx) if mx else None, "reasons": sorted(reasons),
                "samples": len(sm)}


def make_inputs(wl, seed, pinned=False, B=None):
    from styletts2_b200.synthetic import synthetic_batch
    tokens, lengths, bert_dur, noise, ref_s = synthetic_batch(B or wl["B"], wl["N"], wl["model"] == "libritts", seed=seed)
    ts = [tokens, lengths, bert_dur, noise] + ([ref_s] if ref_s is not None else [])
    if pinned:
        ts = [t.pin_memory() for t in ts]
    return ts


DUMP_LIMIT_BYTES = 64 << 20


def dump_outputs(out_dir, arrays):
    """Write what the timed path returned in its last step as DIR/<name>.npy (float32).  An array larger than the budget
    is replaced by a fixed, seeded sample of its elements (<name>.npy) plus the flat indices taken (<name>_index.npy)."""
    import numpy as np
    os.makedirs(out_dir, exist_ok=True)
    budget = DUMP_LIMIT_BYTES // max(1, len(arrays))
    for name, t in arrays.items():
        a = t.detach().float().cpu().numpy()
        if a.nbytes > budget:
            n = budget // 12                      # 4 bytes of value + 8 bytes of index per sampled element
            idx = np.sort(np.random.default_rng(0).choice(a.size, size=n, replace=False)).astype(np.int64)
            np.save(os.path.join(out_dir, f"{name}_index.npy"), idx)
            a = a.reshape(-1)[idx]
        np.save(os.path.join(out_dir, f"{name}.npy"), a)


def kernel_family(name):
    return name.split(" ")[0]


def run_ours(args):
    from styletts2_b200 import lib
    from styletts2_b200 import ops as _ops
    from styletts2_b200.configs import MODEL_CFGS
    from styletts2_b200.inference import Synthesizer
    from styletts2_b200.models import build_model, load_keyed_weights, recursive_munch
    from styletts2_b200.parallel import gather_waveforms, init_from_env, shard_range

    rank, local, world = init_from_env("nccl")
    assert world == args.gpus or world == 1, (world, args.gpus)
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    wl = dict(WORKLOADS[args.workload])
    if args.diffusion_steps:
        wl["steps"] = args.diffusion_steps
    mcfg = MODEL_CFGS[wl["model"]]
    model = build_model(recursive_munch(mcfg))
    for k in model:
        model[k].to(dev).eval()
    load_keyed_weights(model)
    syn = Synthesizer(model, mcfg, dev)
    ms = wl["model"] == "libritts"
    N, T = wl["N"], wl["N"] * wl["fpt"]
    L = 600 * T
    if args.global_batch:
        # strong scaling: ONE global batch, sharded contiguously by utterance (parallel.shard_range), as BASELINE configs[2]/[4]
        gB = args.global_batch
        lo, hi = shard_range(gB, rank, world)
        B = hi - lo
        host_all = make_inputs(wl, seed=1, B=gB)
        host = [t[lo:hi].contiguous().pin_memory() for t in host_all]
        total_utts, scaling = gB, "strong"
    else:
        B = wl["B"]
        host = make_inputs(wl, seed=1 + rank, pinned=True)
        total_utts, scaling = B * world, "weak"
    samples_per_step = total_utts * L
    devin = [t.to(dev) for t in host]
    wav_host = torch.empty(B, L, dtype=torch.float32).pin_memory()
    graph_launches = [0]

    def step(inputs):
        tokens, lengths, bert_dur, noise = inputs[:4]
        ref_s = inputs[4] if ms else None
        if args.graph:
            wav, nl = syn.synthesize_graphed(tokens, lengths, bert_dur, noise, diffusion_steps=wl["steps"], ref_s=ref_s,
                                             pin_frames_per_token=wl["fpt"])
            graph_launches[0] = nl
            return wav
        return syn.synthesize(tokens, lengths, bert_dur, noise, diffusion_steps=wl["steps"], ref_s=ref_s,
                              pin_frames_per_token=wl["fpt"])["wav"]

    def barrier():
        if world > 1:
            torch.distributed.barrier()
        torch.cuda.synchronize()

    def max_over_ranks(v):
        if world == 1:
            return v
        t = torch.tensor([v], device=dev, dtype=torch.float64)
        torch.distributed.all_reduce(t, op=torch.distributed.ReduceOp.MAX)
        return float(t.item())

    def all_ranks(v):
        if world == 1:
            return [v]
        t = torch.zeros(world, device=dev, dtype=torch.float64)
        t[rank] = v
        torch.distributed.all_reduce(t)
        return [float(x) for x in t.tolist()]

    # ---- device-resident throughput (`value`)
    for _ in range(args.warmup):
        step(devin)
    barrier()
    clocks = ClockSampler(local)
    if rank == 0:
        clocks.start()
    n0 = lib.launch_count()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(args.steps):
        wav_last = step(devin)
    e1.record()
    barrier()
    if args.dump_outputs and rank == 0:
        dump_outputs(args.dump_outputs, {"wav": wav_last.view(B, L)})
    launches = lib.launch_count() - n0
    if args.graph:
        launches = graph_launches[0] * args.steps   # kernels of this library inside the replayed CUDA graph x replays
    ms_local = e0.elapsed_time(e1)
    ms_total = max_over_ranks(ms_local)
    per_rank_ms = [v / args.steps for v in all_ranks(ms_local)]
    if args.skip_e2e:
        if rank == 0:
            clocks.stop()
            print(json.dumps({"profile_only": True, "ms_per_step": ms_total / args.steps, "gpu_launches": launches}))
        return
    # ---- end to end through the public API with HOST buffers (`e2e`): H2D of the inputs, the step, D2H of the waveform,
    # and a stream synchronise per step (the caller holds the result before the next request starts)
    def e2e_step():
        ins = [t.to(dev, non_blocking=True) for t in host]
        wav = step(ins)
        wav_host.copy_(wav.view(B, L), non_blocking=True)
        torch.cuda.current_stream().synchronize()
    for _ in range(max(1, args.warmup // 2)):
        e2e_step()
    barrier()
    e2, e3 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e2.record()
    for _ in range(args.steps):
        e2e_step()
    e3.record()
    barrier()
    ms_e2e = max_over_ranks(e2.elapsed_time(e3))
    clk = clocks.stop() if rank == 0 else None
    # ---- optional final collective (the only one on the path): gather the shard waveforms on rank 0 over NCCL
    gather = None
    if args.gather and world > 1:
        wav = step(devin).view(B, L)
        gb = total_utts if args.global_batch else None
        gather_waveforms(wav, world, dst=0, batch=gb)      # untimed: the first collective sets up the NCCL connections
        barrier()
        g0, g1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        g0.record()
        for _ in range(3):
            shards = gather_waveforms(wav, world, dst=0, batch=gb)
        g1.record()
        barrier()
        gms = max_over_ranks(g0.elapsed_time(g1)) / 3
        if rank == 0:
            nbytes = sum(s.numel() * 4 for s in shards)
            gather = {"bytes": nbytes, "ms": gms, "gbs": nbytes / (gms / 1e3) / 1e9, "shards": [int(s.shape[0]) for s in shards]}

    # ---- per-launch profile: consecutive eager passes with CUDA events around every profiled launch (the first pass is
    # discarded; the passes run back to back, i.e. in the same sustained regime as the timed loop)
    tokens, lengths, bert_dur, noise = devin[:4]
    kw = dict(diffusion_steps=wl["steps"], ref_s=devin[4] if ms else None, pin_frames_per_token=wl["fpt"])
    passes = []
    stage_ms = {}
    for i in range(1 + args.profile_passes):
        _ops.PROFILE = []
        mk = []
        syn.synthesize(tokens, lengths, bert_dur, noise, stage_marks=mk, **kw)
        torch.cuda.synchronize()
        prof, _ops.PROFILE = _ops.PROFILE, None
        if i == 0:
            continue
        passes.append([(n_, f_, b_, a_.elapsed_time(z_), m_) for n_, f_, b_, a_, z_, m_ in prof])
        for (_, ea), (nb, eb) in zip(mk[:-1], mk[1:]):
            stage_ms[nb] = stage_ms.get(nb, 0.0) + ea.elapsed_time(eb) / args.profile_passes
    if rank != 0:
        torch.distributed.barrier()
        torch.distributed.destroy_process_group()
        return
    rows = {}
    for p_ in passes:
        for n_, f_, b_, t_, m_ in p_:
            r_ = rows.setdefault(n_, dict(n=0, ms=0.0, flops=0.0, bytes=0.0, exec_flops=0.0))
            r_["n"] += 1; r_["ms"] += t_; r_["flops"] += f_; r_["bytes"] += b_; r_["exec_flops"] += f_ * m_
    for r_ in rows.values():
        for k_ in ("n", "ms", "flops", "bytes", "exec_flops"):
            r_[k_] /= len(passes)
    eager_ms = sum(stage_ms.values())
    ms_per_step = ms_total / args.steps
    fam = {}
    for n_, r_ in rows.items():
        f_ = fam.setdefault(kernel_family(n_), dict(n=0, ms=0.0, flops=0.0, bytes=0.0, exec_flops=0.0))
        for k_ in f_:
            f_[k_] += r_[k_]
    hbm_peak, tc_peak, tc_burst, peak_src = measured_peaks()
    # dominant kernel = the tensor-core conv (Conv1d + polyphase ConvTranspose1d launches of tc::conv1d_tc_kernel)
    tc = dict(n=0, ms=0.0, flops=0.0, bytes=0.0, exec_flops=0.0)
    for k_ in ("conv1d_tc", "convT_tc"):
        for kk in tc:
            tc[kk] += fam.get(k_, {}).get(kk, 0.0)
    # the eager profile pass has launch gaps the graph replay does not: scale the kernel's time by its SHARE of the step
    share = tc["ms"] / eager_ms if eager_ms else 0.0
    tc_ms_sustained = share * ms_per_step if args.graph else tc["ms"]
    n_tc = max(1.0, tc["n"])
    alg_tflops = tc["flops"] / (tc["ms"] / 1e3) / 1e12 if tc["ms"] else 0.0
    exe_tflops = tc["exec_flops"] / (tc["ms"] / 1e3) / 1e12 if tc["ms"] else 0.0
    traffic = ncu_traffic()
    hbm_kernels = {}
    for k_ in ("istft20", "sine_source", "stft20", "instance_stats", "adain_lrelu_pool", "conv1d_simt"):
        if k_ in fam and fam[k_]["ms"] > 0:
            f_ = fam[k_]
            hbm_kernels[k_] = {"launches": f_["n"], "ms": round(f_["ms"], 4), "algorithmic_gbs": round(f_["bytes"] / (f_["ms"] / 1e3) / 1e9, 1),
                               "frac_of_hbm_peak": round(f_["bytes"] / (f_["ms"] / 1e3) / 1e9 / hbm_peak, 3)}
    den = {}
    if "linear_tc" in fam:
        f_ = fam["linear_tc"]
        att = dict(ms=0.0, flops=0.0)
        for k_ in ("attention", "attention_tc"):
            for kk in att:
                att[kk] += fam.get(k_, {}).get(kk, 0.0)
        den = {"linear_tc_ms": round(f_["ms"], 3), "linear_tc_fp32_tflops": round(f_["flops"] / (f_["ms"] / 1e3) / 1e12, 1),
               "linear_tc_executed_tflops": round(f_["exec_flops"] / (f_["ms"] / 1e3) / 1e12, 1),
               "attention_ms": round(att["ms"], 3),
               "attention_fp32_tflops": round(att["flops"] / (att["ms"] / 1e3) / 1e12, 1) if att["ms"] else None,
               "sampler_ms": round(stage_ms.get("sampler", 0.0), 3),
               "sampler_algorithmic_tflops": round(denoiser_flops(N, wl["steps"]) * B / (stage_ms.get("sampler", 1e9) / 1e3) / 1e12, 1),
               "flops_per_utt_eval": 37.8e6 * N + 6144.0 * N * N, "evals": 2 * (wl["steps"] - 1)}
    if args.dump_launches:
        out_rows = [dict(launch=k_, n=round(v_["n"], 1), ms=round(v_["ms"], 4),
                         fp32_tflops=round(v_["flops"] / (v_["ms"] / 1e3) / 1e12, 1) if v_["ms"] else None,
                         executed_tflops=round(v_["exec_flops"] / (v_["ms"] / 1e3) / 1e12, 1) if v_["ms"] else None,
                         algorithmic_gbs=round(v_["bytes"] / (v_["ms"] / 1e3) / 1e9, 1) if v_["ms"] else None)
                    for k_, v_ in sorted(rows.items(), key=lambda kv: -kv[1]["ms"])]
        with open(args.dump_launches, "w") as f_:
            json.dump(out_rows, f_, indent=1)
    value = samples_per_step / (ms_per_step / 1e3)
    e2e_value = samples_per_step / (ms_e2e / args.steps / 1e3)
    h2d = sum(t.numel() * t.element_size() for t in host)
    d2h = wav_host.numel() * 4
    dec_ms = stage_ms.get("decoder", 0.0)
    alg_bytes = VOCODER_BYTES_PER_FRAME[wl["model"]] * B * T + VOCODER_WEIGHT_BYTES[wl["model"]]
    alg_flops = VOCODER_FLOPS_PER_FRAME[wl["model"]] * B * T
    line = {
        "metric": "24 kHz waveform samples/sec", "value": value, "unit": "samples/s", "n_gpus": world, "steps": args.steps,
        "warmup": args.warmup, "ms_per_step": ms_per_step, "higher_is_better": True, "scaling": scaling, "vs_baseline": None,
        "dtype": "f32", "data": "synthetic (key-seeded random weights, seeded tokens/bert_dur/noise; durations pinned to 4 frames/token)",
        "config": {"workload": f"{args.workload}: {wl['desc']}", "per_gpu_batch": B, "global_batch": total_utts, "tokens": N, "frames": T,
                   "samples_per_utt": L, "diffusion_steps": wl["steps"],
                   "sharding": f"utterances over {world} rank(s) ({'one global batch split by shard_range' if args.global_batch else 'same batch per rank'}), no data-path collective",
                   "l2": "inputs+activations per step (>3 GB) exceed the 50 MB L2; no flush needed",
                   "launch": "one CUDA graph per step" if args.graph else "eager"},
        "e2e": {"value": e2e_value, "unit": "samples/s", "h2d_bytes_per_step": h2d, "d2h_bytes_per_step": d2h,
                "sync": "stream synchronise after every step's D2H copy"},
        "gpu_launches": launches,
        "per_rank_ms_per_step": per_rank_ms,
        "stages_ms": {k_: round(v_, 3) for k_, v_ in stage_ms.items()},
        "clocks": clk,
        "roofline": {"kernel": "st2::tc::conv1d_tct_kernel (time-major, Cout <= 128) + st2::tc::conv1d_tc_kernel (channel-major, Cout >= 256): wgmma "
                               "implicit-GEMM Conv1d / polyphase ConvTranspose1d, fp16 high planes + e4m3 correction MMA, 2 MMA-times per fp32 "
                               "product; 3 in the F0/N predictor",
                     "bound": "tensor", "achieved": alg_tflops, "peak": tc_peak, "unit": "TFLOP/s", "frac": alg_tflops / tc_peak,
                     "frac_algorithmic": alg_tflops / tc_peak, "frac_executed": exe_tflops / tc_peak, "executed_tflops": exe_tflops,
                     "traffic": (traffic or {}).get("dram_bytes_per_launch"), "traffic_source": (traffic or {}).get("source"),
                     "peak_source": peak_src, "peak_burst": tc_burst, "launches_per_step": tc["n"],
                     "avg_launch_ms": tc["ms"] / n_tc, "algorithmic_gflop_per_launch": tc["flops"] / n_tc / 1e9,
                     "algorithmic_bytes_per_launch": tc["bytes"] / n_tc,
                     "hbm_algorithmic_gbs": tc["bytes"] / (tc["ms"] / 1e3) / 1e9 if tc["ms"] else None, "hbm_peak_gbs": hbm_peak,
                     "kernel_ms_per_step_eager_events": tc["ms"], "kernel_share_of_step": share,
                     "kernel_ms_per_step_sustained": tc_ms_sustained,
                     "achieved_sustained": tc["flops"] / (tc_ms_sustained / 1e3) / 1e12 if tc_ms_sustained else None,
                     "decoder_ms_per_step": dec_ms, "eager_step_ms": eager_ms,
                     "vocoder_path_algorithmic": {"bytes_per_step": alg_bytes, "flops_per_step": alg_flops,
                                                  "gbs": alg_bytes / (dec_ms / 1e3) / 1e9 if dec_ms else None,
                                                  "tflops": alg_flops / (dec_ms / 1e3) / 1e12 if dec_ms else None},
                     "hbm_bound_kernels": hbm_kernels, "denoiser": den,
                     "note": "achieved = ALGORITHMIC fp32 FLOPs (2*Cin*Cout*K*L*B summed over the step's launches of the kernel) / CUDA-event "
                             f"time of those launches, mean of {args.profile_passes} back-to-back eager passes after a discarded one; "
                             "frac_executed counts the MMAs actually issued (2 or 3 per product); kernel_ms_per_step_sustained = the kernel's "
                             "share of the eager pass x the graph-replayed step time"},
    }
    if gather:
        line["gather"] = gather
    if args.cpu_baseline:
        line["cpu_baseline"] = cpu_reference(wl, sample_B=args.cpu_batch, steps=3, warmup=1)
    print(json.dumps(line))
    if world > 1:
        torch.distributed.barrier()
        torch.distributed.destroy_process_group()


def cpu_reference(wl, sample_B, steps, warmup, probe=True):
    """The reference algorithm (oracle port, torch CPU fp32) on the host cores, bounded sample of the workload.
    The port is pinned against the original implementation
    (tests/golden/PINNING*.json).  Thread count: a short probe at 8 / 32 / all cores picks the fastest."""
    sys.path.insert(0, os.path.join(ROOT, "oracle"))
    import styletts2_oracle as O
    from styletts2_b200.configs import MODEL_CFGS
    from styletts2_b200.synthetic import keyed_state_dict

    mcfg = MODEL_CFGS[wl["model"]]
    shapes = json.load(open(os.path.join(ROOT, "tests", "golden", f"state_shapes_{wl['model']}.json")))
    sds = {k: keyed_state_dict({n: tuple(s) for n, s in shapes[k].items()}, k) for k in shapes}

    def run(Bs, n_run):
        sub = dict(wl, B=Bs)
        ins = make_inputs(sub, seed=1)
        tokens, lengths, bert_dur, noise = ins[:4]
        ref_s = ins[4] if wl["model"] == "libritts" else None
        forced = torch.full((Bs, wl["N"]), float(wl["fpt"]))
        ts, nsamp = [], 0
        for _ in range(n_run):
            t0 = time.time()
            with torch.no_grad():
                out = O.synthesize(sds, mcfg, tokens, lengths, bert_dur, noise, diffusion_steps=wl["steps"], ref_s=ref_s,
                                   forced_durations=forced)
            ts.append(time.time() - t0)
            nsamp = out["wav"].numel()
        return ts, nsamp

    ncpu = os.cpu_count() or 1
    probe_res = {}
    best = min(32, ncpu)
    if probe:
        # one utterance per thread count (bounded: the probe must not eat the few minutes the default run has; all 128
        # threads of the GPU box were measured 7x slower than 8 in round 1 -- oversubscribed intra-op pools -- and are
        # probed only up to 64)
        for nt in sorted({min(8, ncpu), min(16, ncpu), min(32, ncpu), min(64, ncpu)}):
            torch.set_num_threads(nt)
            ts, ns = run(1, 1)
            probe_res[nt] = round(ns / ts[-1])
        best = max(probe_res, key=probe_res.get)
    torch.set_num_threads(best)
    ts, nsamp = run(sample_B, warmup + steps)
    ts = ts[warmup:]
    med = statistics.median(ts)
    return {"value": nsamp / med, "unit": "samples/s", "cores": best, "host_cores": ncpu, "kind": "port",
            "thread_probe_samples_per_s": probe_res,
            "sample": f"{sample_B} utterance(s) of the workload ({wl['N']} tokens, {wl['N'] * wl['fpt']} frames, K={wl['steps']}), "
                      f"{warmup} warm-up + {len(ts)} timed runs (median), torch {torch.__version__} CPU, {best} of {ncpu} threads "
                      f"(fastest of the probe); oracle port of the reference forward",
            "seconds_per_run": med, "runs_s": [round(t, 3) for t in ts]}


def run_reference(args):
    rank = int(os.environ.get("RANK", "0"))
    if rank != 0:
        return
    wl = dict(WORKLOADS[args.workload])
    if args.diffusion_steps:
        wl["steps"] = args.diffusion_steps
    cb = cpu_reference(wl, sample_B=args.cpu_batch, steps=args.steps, warmup=args.warmup)
    line = {"impl": "reference", "metric": "24 kHz waveform samples/sec", "value": cb["value"], "unit": "samples/s",
            "n_gpus": args.gpus, "steps": args.steps, "warmup": args.warmup, "ms_per_step": cb["seconds_per_run"] * 1e3,
            "higher_is_better": True, "scaling": "weak", "vs_baseline": None, "dtype": "f32", "data": "synthetic",
            "config": {"workload": f"{args.workload}: {wl['desc']} (bounded sample: {args.cpu_batch} utterance(s) per step)"},
            "cpu_baseline": cb, "e2e": {"value": cb["value"], "unit": "samples/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0},
            "gpu_launches": 0}
    print(json.dumps(line))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--impl", default="ours", choices=["ours", "reference"])
    ap.add_argument("--workload", default="C2", choices=list(WORKLOADS))
    ap.add_argument("--global-batch", type=int, default=0, help="shard ONE batch of this many utterances over the ranks (strong scaling)")
    ap.add_argument("--diffusion-steps", type=int, default=0, help="override the workload's sampler steps (C5 sweep: 3/5/10/50)")
    ap.add_argument("--gather", action="store_true", help="N>1: time the optional final NCCL gather of the waveforms on rank 0")
    ap.add_argument("--cpu-batch", type=int, default=2)
    ap.add_argument("--profile-passes", type=int, default=3)
    ap.add_argument("--no-cpu-baseline", dest="cpu_baseline", action="store_false")
    ap.add_argument("--no-graph", dest="graph", action="store_false", help="eager launches instead of one CUDA graph per step")
    ap.add_argument("--dump-launches", default=None, help="write the per-shape launch table (CUDA events, eager passes) to this JSON file")
    ap.add_argument("--dump-outputs", default=None, metavar="DIR",
                    help="write the waveforms of the last timed step as DIR/<name>.npy (float32, at most 64 MB; seeded inputs)")
    ap.add_argument("--skip-e2e", action="store_true", help="profiling runs only (ncu): device-resident loop, no JSON contract line")
    args = ap.parse_args()
    if args.impl == "reference":
        run_reference(args)
    else:
        run_ours(args)


if __name__ == "__main__":
    main()
