#!/usr/bin/env python
"""BSS Eval v4 of source images (ctn_bss_eval_images, museval's `eval_mus_track` in fp64 on the GPU) at MUSDB18 size: one JSON line.

    python tools/bench_museval.py [--reps 5] [--warmup 1] [--no-oracle] [--profile DIR] [--out result.json]

Synthetic track: 4 stems plus their sum as accompaniment, stereo, 44.1 kHz, 60 s and 240 s; low-pass filtered noise references,
estimates FIR(reference) + cross-talk + noise (tests/museval_ref.py).  eval_track makes museval's two calls: the 4 stems
(J = 4, I = 2, a 4096 x 4096 Gram matrix) and vocals / accompaniment (J = 2).  Per track length, the median (min, max) of `reps`
repetitions after `warmup`, each bracketed by CUDA events and ended by a synchronise:
  call_ms[J]      the C call alone (no host synchronisation inside), for each of the two calls
  eval_track_ms   eval_track from host numpy arrays: copies, both calls, status reads and results back to numpy
  launches, workspace_bytes   per call
  oracle_s        the fp64 numpy / scipy oracle (tests/museval_ref.py; not museval itself) on the CPU, both calls, 60 s only
  worst_err_db    largest |GPU - oracle| over the finite values of that run
solve_ms: at N = 4096 with 8 right-hand sides, the all-columns solve against the one-CTA-per-column solve of bss_eval_sources on
the same factor.  --profile DIR: a separate torch.profiler run of one 60 s eval_track, CUDA time per kernel and per stage.
The card's name and power limit are read in the same run; no device setting is changed."""
import argparse
import collections
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "dnn-based_source_separation_b200"))
sys.path.insert(0, os.path.join(ROOT, "tests"))

import museval_ref as R  # noqa: E402
from ctn_b200 import _native as N  # noqa: E402
from ctn_b200.utils import museval as MV  # noqa: E402

SR = 44100
NAMES = ["vocals", "drums", "bass", "other"]
STAGES = (("silence", ("k_mus_silent",)), ("correlations", ("k_mus_corr", "k_mus_combine", "k_mus_build")),
          ("cholesky", ("k_chol_",)), ("solve", ("k_mus_fwd_step", "k_mus_bwd_step")), ("projection", ("k_mus_project",)),
          ("finish", ("k_mus_finish",)))


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i",
                          str(torch.cuda.current_device())], capture_output=True, text=True, check=True).stdout.strip()
    return [s.strip() for s in out.split(",")]


def median_ms(fn, reps, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    times = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        times.append(a.elapsed_time(b))
    times.sort()
    return times[len(times) // 2], times[0], times[-1]


def track(seconds):
    refs, ests = R.make_track(np.random.default_rng(seconds), 4, 2, seconds * SR, coloured=True)
    references = {k: refs[i].T for i, k in enumerate(NAMES)}
    estimates = {k: ests[i].T for i, k in enumerate(NAMES)}
    references["accompaniment"] = (refs[1] + refs[2] + refs[3]).T
    estimates["accompaniment"] = (ests[1] + ests[2] + ests[3]).T
    return references, estimates


def call_case(ref_h, est_h, reps, warmup):
    """the C call alone on device tensors (J, I, T)"""
    ref, est = torch.from_numpy(ref_h).cuda(), torch.from_numpy(est_h).cuda()
    J, I, T = ref.shape
    nbytes = C.c_size_t(0)
    N.check(N.ctn_bss_images_workspace_bytes(J, I, T, SR, SR, C.byref(nbytes)))
    ws = torch.empty(nbytes.value + 256, dtype=torch.uint8, device="cuda")
    base, avail = N.aligned(ws)
    nwin = R.nwin_of(T, SR, SR)
    outs = [torch.empty((J, nwin), dtype=torch.float64, device="cuda") for _ in range(4)]
    status = torch.empty(1, dtype=torch.int32, device="cuda")
    st = N.stream_ptr(ref.device)

    def call():
        N.check(N.ctn_bss_eval_images(ref.data_ptr(), est.data_ptr(), J, I, T, SR, SR, *(t.data_ptr() for t in outs), status.data_ptr(),
                                      base, avail, st), "ctn_bss_eval_images")

    ms = median_ms(call, reps, warmup)
    launches = N.ctn_last_launch_count()
    assert int(status) == 0
    return {"J": J, "I": I, "T": T, "call_ms": ms[0], "call_ms_min_max": ms[1:], "launches": launches,
            "workspace_bytes": nbytes.value}


def stack(d, names):
    return np.stack([np.asarray(d[k]).T for k in names]).astype(np.float32)


def run_track(seconds, reps, warmup, oracle):
    references, estimates = track(seconds)
    calls = [call_case(stack(references, NAMES), stack(estimates, NAMES), reps, warmup),
             call_case(stack(references, ["vocals", "accompaniment"]), stack(estimates, ["vocals", "accompaniment"]), reps, warmup)]
    torch.cuda.empty_cache()
    ms = median_ms(lambda: MV.eval_track(references, estimates, SR), reps, warmup)
    res = {"seconds": seconds, "calls": calls, "eval_track_ms": ms[0], "eval_track_ms_min_max": ms[1:]}
    if oracle:
        scores = MV.eval_track(references, estimates, SR)
        t0 = time.perf_counter()
        four = R.metrics(stack(references, NAMES), stack(estimates, NAMES), SR, SR)
        two = R.metrics(stack(references, ["vocals", "accompaniment"]), stack(estimates, ["vocals", "accompaniment"]), SR, SR)
        res["oracle_s"] = time.perf_counter() - t0
        worst = 0.0
        for names, o, skip in ((NAMES, four, "vocals"), (["vocals", "accompaniment"], two, None)):
            for i, k in enumerate(names):
                if k == skip:
                    continue
                for q, m in enumerate(MV.METRICS):
                    fin = np.isfinite(o[q][i])
                    worst = max(worst, float(np.max(np.abs(scores[k][m][fin] - o[q][i][fin]))))
        res["worst_err_db"] = worst
    return res


_p, _i = C.c_void_p, C.c_int
probe_factor = N._sig("ctn_probe_chol_factor", _i, _p, _p, _p, _i, _i, _p)
probe_solve = N._sig("ctn_probe_chol_solve", _i, _p, _p, _p, _p, _i, _i, _i, _i, _p)


def solve_case(reps, warmup, n=4096, nrhs=8):
    rng = np.random.default_rng(7)
    X = torch.from_numpy(rng.standard_normal((n + 600, n))).cuda()
    A = (X.T @ X / n).contiguous()
    del X
    W = torch.empty((n // 64, 64, 64), dtype=torch.float64, device="cuda")
    flag = torch.empty(1, dtype=torch.int32, device="cuda")
    N.check(probe_factor(A.data_ptr(), W.data_ptr(), flag.data_ptr(), n, 1, None))
    B = torch.from_numpy(rng.standard_normal((n, nrhs))).cuda()
    rows, tmp, cols = B.clone(), torch.empty_like(B), B.T.contiguous()

    def multi():
        rows.copy_(B)
        N.check(probe_solve(A.data_ptr(), W.data_ptr(), rows.data_ptr(), tmp.data_ptr(), n, 1, nrhs, 1, None))

    def percol():
        cols.copy_(B.T)
        N.check(probe_solve(A.data_ptr(), W.data_ptr(), cols.data_ptr(), None, n, 1, nrhs, 0, None))

    m, c = median_ms(multi, reps, warmup), median_ms(percol, reps, warmup)
    diff = float((rows - cols.T).abs().max() / rows.abs().max())
    return {"N": n, "nrhs": nrhs, "all_columns_ms": m[0], "per_column_ms": c[0], "rel_diff": diff}


def profile(outdir):
    from torch.profiler import ProfilerActivity, profile as prof
    references, estimates = track(60)
    MV.eval_track(references, estimates, SR)
    torch.cuda.synchronize()
    with prof(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as p:
        MV.eval_track(references, estimates, SR)
        torch.cuda.synchronize()
    kernels = collections.Counter()
    counts = collections.Counter()
    for e in p.key_averages():
        if e.device_type == torch.autograd.DeviceType.CUDA or getattr(e, "self_device_time_total", 0) > 0:
            t = getattr(e, "self_device_time_total", None) or getattr(e, "self_cuda_time_total", 0)
            kernels[e.key] += t / 1e3
            counts[e.key] += e.count
    stages = collections.Counter()
    for k, t in kernels.items():
        for s, keys in STAGES:
            if any(x in k for x in keys):
                stages[s] += t
                break
        else:
            stages["other"] += t
    os.makedirs(outdir, exist_ok=True)
    with open(os.path.join(outdir, "museval_profile.txt"), "w") as f:
        f.write(p.key_averages().table(sort_by="self_cuda_time_total", row_limit=40))
    return {"stage_ms": dict(stages), "top_kernels_ms": {k: round(v, 3) for k, v in kernels.most_common(12)},
            "top_kernel_counts": {k: counts[k] for k, _ in kernels.most_common(12)}}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--no-oracle", action="store_true")
    ap.add_argument("--profile", default=None)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_museval.py measures the GPU path and needs a CUDA device")
    name, power, clock = card()
    res = {"device": name, "power_limit": power, "max_sm_clock": clock}
    if a.profile:
        res["profile_60s"] = profile(a.profile)
    else:
        res["tracks"] = [run_track(s, a.reps, a.warmup, s == 60 and not a.no_oracle) for s in (60, 240)]
        res["solve"] = solve_case(a.reps, a.warmup)
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
