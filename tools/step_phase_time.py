"""Where a tile's time goes inside the fused hidden-32 step (k_step_fused), phase by phase.

Runs bench.py's flagship workload (20 objects x 1200 rays x 10 samples, hidden 32, the same parameter and batch seeds
as its device-resident arm) through vmb_step_trace: the same step, launched from the phase-stamped instantiation
(thread 0 of each warpgroup reads clock64() at every phase boundary of each tile, and %globaltimer at kernel entry,
after its last segment, at the start of the finish and at exit).  The traced steps run back to back, each into its
own trace buffer, with a CUDA event between consecutive launches.  Prints one JSON line: the median cycles of each
phase per tile and its share of the tile, the prologue / segment-flush / wait / finish cycles, the timeline of a step
(event time, kernel span on %globaltimer, CTA entry skew, the busiest CTA's tile cycles and its cycles from the last
segment to exit, event time minus span = launch and drain, the SM clock the kernel ran at = cycles over
%globaltimer time), the observed %globaltimer resolution, and the card's name, power limit and SM clock read while
the traced steps run.

    python tools/step_phase_time.py [--steps 50] [--warmup 10]
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import threading

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

from vmap_b200 import _lib  # noqa: E402
from vmap_b200 import synth as vo  # noqa: E402
from vmap_b200.ensemble import StepInputs, VmapEnsemble  # noqa: E402

B, R, S, HIDDEN = 20, 1200, 10, 32                      # bench.py N_OBJ, N_RAYS, N_SAMPLES, HIDDEN
# row layout of the trace (uf::TR_* in k_step_fused.cuh, VMB_TRACE_STRIDE in vmap_b200.h)
TR_HDR, TR_NST, TR_TILES = 16, 20, 64
TR_STRIDE = TR_HDR + TR_TILES * TR_NST
MAX_CTAS = 192
PHASES = ("pe_forward", "in_layer", "mid1", "cat_layer", "mid2", "color_linear_alpha", "out_color",
          "heads_transpose", "render_loss", "d_hc", "d_fc4", "d_fc3", "d_fc2", "d_fc1", "d_emb",
          "eg_store", "pe_backward", "dB")


def gpu_info():
    q = "name,power.limit,clocks.max.sm"
    r = subprocess.run(["nvidia-smi", "-i", str(torch.cuda.current_device()), f"--query-gpu={q}",
                        "--format=csv,noheader,nounits"], capture_output=True, text=True, timeout=30)
    f = [x.strip() for x in r.stdout.strip().split(",")]
    return {"name": f[0], "power_limit_w": float(f[1]), "sm_max_mhz": float(f[2])}


class SmClock:
    """nvidia-smi's SM clock, sampled every 50 ms while the traced steps run; the poller is stopped in stop()."""

    def __init__(self):
        self.vals, self.proc = [], None

    def start(self):
        self.proc = subprocess.Popen(["nvidia-smi", "-i", str(torch.cuda.current_device()), "--query-gpu=clocks.sm",
                                      "--format=csv,noheader,nounits", "-lms", "50"],
                                     stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True)
        threading.Thread(target=self._pump, daemon=True).start()

    def _pump(self):
        for ln in self.proc.stdout:
            try:
                self.vals.append(float(ln.strip()))
            except ValueError:
                pass

    def stop(self):
        if self.proc is not None and self.proc.poll() is None:
            self.proc.terminate()
            self.proc.wait()
        v = sorted(self.vals)
        return v[len(v) // 2] if v else None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=50, help="traced steps")
    ap.add_argument("--warmup", type=int, default=10)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("step_phase_time.py needs a CUDA device")
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    L = _lib.lib()

    ens = VmapEnsemble(B, hidden=HIDDEN, scale=2.0, device=dev, impl="umma")
    ens.load_stacked(vo.init_params(B, HIDDEN, seed=1000))
    pool = [StepInputs(B, R, S, device=dev).copy_from(StepInputs(B, R, S).fill(vo.synthetic_batch(B, R, S, seed=i)),
                                                      non_blocking=False) for i in range(8)]
    for i in range(args.warmup):
        ens.step(pool[i % len(pool)].views)

    n_sm = torch.cuda.get_device_properties(dev).multi_processor_count
    rows = 2 * min(n_sm, MAX_CTAS)
    traces = torch.zeros(args.steps, rows * TR_STRIDE, dtype=torch.int64, device=dev)
    loss_out = torch.zeros(1, dtype=torch.float32, device=dev)
    stream = C.c_void_p(torch.cuda.current_stream().cuda_stream)

    def traced_step(i, trace):
        a = ens._step_args(pool[i % len(pool)].views, True, fuse_adam=True, loss_out=loss_out)
        with torch.cuda.device(dev):
            _lib.check(ens._handle, L.vmb_step_trace(ens._handle, C.byref(a), C.c_void_p(trace.data_ptr()),
                                                     trace.numel(), stream), "vmb_step_trace")
        ens.step_count += 1

    for i in range(3):                                   # warm the traced instantiation
        traced_step(args.warmup + i, traces[0])
    traces.zero_()
    torch.cuda.synchronize()

    ev = [torch.cuda.Event(enable_timing=True) for _ in range(args.steps + 1)]
    clock = SmClock()
    clock.start()
    try:
        for i in range(args.steps):                      # back to back: the host enqueues faster than a step runs
            ev[i].record()
            traced_step(args.warmup + 3 + i, traces[i])
        ev[args.steps].record()
        torch.cuda.synchronize()
    finally:
        sm_mhz = clock.stop()
    ens.check_status()

    tiles, prologue, flush, wait, finish, kernel = [], [], [], [], [], []
    tl = {k: [] for k in ("event_us", "span_us", "entry_skew_us", "busiest_tile_cycles", "busiest_last_seg_to_exit_cycles",
                          "wait_cycles_p10", "wait_cycles_p50", "wait_cycles_p90", "wait_cycles_max",
                          "finish_cycles_p50", "finish_cycles_max", "event_minus_span_us", "sm_mhz_from_trace")}
    gt_res = []
    all_t = traces.view(args.steps, rows, TR_STRIDE).cpu().numpy().astype(np.int64)
    for i in range(1, args.steps):                       # step 0 follows the warm-up's synchronise: not back to back
        t = all_t[i]
        ctas = [r for r in t[0::2] if r[4] != 0]         # warpgroup 0's row of every CTA that ran
        cta_tiles, cta_tail, cta_wait, cta_fin = [], [], [], []
        for r in t:
            if r[4] == 0:                                # no CTA ran this row
                continue
            nt = int(min(r[5], TR_TILES))
            st = r[TR_HDR:TR_HDR + nt * TR_NST].reshape(nt, TR_NST)[:, :len(PHASES) + 1]
            tiles.append(np.diff(st, axis=1))
            if nt:
                prologue.append(st[0, 0] - r[0])
            if r[7]:
                flush.append(r[6] / r[7])
        for r in ctas:
            nt = int(min(r[5], TR_TILES))
            st = r[TR_HDR:TR_HDR + nt * TR_NST].reshape(nt, TR_NST)
            cta_tiles.append(int((st[:, len(PHASES)] - st[:, 0]).sum()) if nt else 0)
            cta_tail.append(r[4] - r[2])
            cta_wait.append(r[12])
            cta_fin.append(r[4] - r[3])
            kernel.append(r[4] - r[0])
        wait += cta_wait
        finish += cta_fin
        g = np.array([[r[8], r[9], r[10], r[11]] for r in ctas], np.int64)
        d = np.diff(np.unique(g))
        gt_res.append(int(d[d > 0].min()) if (d > 0).any() else 0)
        span = (g[:, 3].max() - g[:, 0].min()) / 1e3
        ev_us = ev[i].elapsed_time(ev[i + 1]) * 1e3
        busiest = int(np.argmax(cta_tiles))
        w = np.array(cta_wait, np.float64)
        tl["event_us"].append(ev_us)
        tl["span_us"].append(span)
        tl["entry_skew_us"].append((g[:, 0].max() - g[:, 0].min()) / 1e3)
        tl["busiest_tile_cycles"].append(cta_tiles[busiest])
        tl["busiest_last_seg_to_exit_cycles"].append(cta_tail[busiest])
        for q in (10, 50, 90):
            tl[f"wait_cycles_p{q}"].append(float(np.percentile(w, q)))
        tl["wait_cycles_max"].append(float(w.max()))
        tl["finish_cycles_p50"].append(float(np.median(cta_fin)))
        tl["finish_cycles_max"].append(float(np.max(cta_fin)))
        tl["event_minus_span_us"].append(ev_us - span)
        # the SM clock the kernel ran at: each CTA's clock64 cycles over its %globaltimer nanoseconds, entry to exit
        tl["sm_mhz_from_trace"].append(float(np.median([(r[4] - r[0]) / (r[11] - r[8]) * 1e3 for r in ctas])))

    ph = np.concatenate(tiles, axis=0)
    tile_tot = ph.sum(axis=1)
    share = ph.sum(axis=0) / tile_tot.sum()
    med = np.median(ph, axis=0)
    kern_cyc = float(np.median(kernel))
    line = {
        "tool": "step_phase_time", "kernel": "k_step_fused<10, false, true> (phase-stamped)",
        "workload": f"{B} objects x {R} rays x {S} samples, hidden {HIDDEN} (bench.py device-resident arm)",
        "gpu": dict(gpu_info(), sm_mhz_during_trace=sm_mhz),
        "steps": args.steps, "tiles_sampled": int(ph.shape[0]),
        "tile_cycles_median": float(np.median(tile_tot)),
        "phases": {n: {"median_cycles": float(m), "share": round(float(s), 4)} for n, m, s in zip(PHASES, med, share)},
        "prologue_cycles_median": float(np.median(prologue)),
        "segment_flush_cycles_median": float(np.median(flush)),
        "wait_cycles_median": float(np.median(wait)),       # grid barrier, or the readiness waits of the finish
        "finish_cycles_median": float(np.median(finish)),   # finish start -> exit, waits included
        "kernel_cycles_median": kern_cyc,
        "kernel_us_at_sm_clock": kern_cyc / sm_mhz if sm_mhz else None,
        # per-step timeline, median over the traced steps
        "timeline_median": {k: float(np.median(v)) for k, v in tl.items()},
        "globaltimer_resolution_ns": int(min(x for x in gt_res if x > 0)) if any(gt_res) else None,
    }
    print(json.dumps(line))


if __name__ == "__main__":
    main()
