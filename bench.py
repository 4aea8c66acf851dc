#!/usr/bin/env python
"""bench.py — SLAM+NeRF frames/sec on the synthetic 640x480 stream (BASELINE.json metric).

  python bench.py [--gpus N] [--steps K] [--warmup W] [--impl ours|reference] [--dump-outputs DIR]
  python -m torch.distributed.run --nnodes=1 --nproc-per-node N --master-addr 127.0.0.1 ... bench.py --gpus N ...

A STEP = one input frame of the procedural Replica-shaped stream (BASELINE.json configs[1]:
640x480, buffer=100, --slam --fusion=nerf) pushed through RaftVisualFrontend.forward (feature
encoder, motion filter, and on keyframes: proximity edges, correlation volumes, 4+2 update
iterations of {reproject, 4-level lookup, update operator, 2 BA iterations, upsampling}), with
`--nerf-iters` NeRF training iterations (2^18 samples each) issued per frame on a second stream
(N == 1) or on the trainer ranks (N > 1; rank 0 = SLAM, ranks 1.. = data-parallel NeRF).
An untimed PRIMING phase first brings the system to steady state (SLAM initialised, NeRF holds
keyframes) — it is state preparation, like building a model, and is reported in config.

  value  frames/s with the stream already resident in HBM (device tensors)
  e2e    frames/s through the public API with HOST (pinned) frames: H2D of every frame inside the
         timed region + D2H read of the step's result (current pose + NeRF loss)
Timing: CUDA events on the launching streams + barrier/synchronize, max over ranks.  Inputs of a
step (the frame, 1.2 MB) are new every step and the per-keyframe working set (correlation
pyramids ~80 MB/edge, NeRF sample buffers) exceeds L2, so no explicit L2 flush is needed
(config.l2 says so).
"""
import argparse
import json
import os
import subprocess
import sys
import threading
import time
import types

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

W_IMG, H_IMG = 640, 480
STREAM_STEP = 0.035           # camera pace: ~every 3rd-4th frame becomes a keyframe
NERF_SM_BUDGET_SHARED = 64    # SMs of the persistent NeRF kernels when SLAM and NeRF share one GPU (N = 1): about half
# --workload: cfg2 = BASELINE.json configs[1] (the metric's configuration, default); cfg5 = configs[4]'s shapes
# (1280x720, buffer 200); cfg4 = configs[3] (640x480, buffer 400, plus the global-BA / alt-corr pass over the filled
# window, timed separately as `global_ba`).
WORKLOADS = {"cfg2": dict(w=640, h=480, buffer=100, corr_slots=112, name="configs[1]: Replica-office0-shaped synthetic 640x480"),
             "cfg4": dict(w=640, h=480, buffer=400, corr_slots=112, name="configs[3]: long synthetic 640x480 trajectory, buffer=400, global BA on the alt-corr path"),
             "cfg5": dict(w=1280, h=720, buffer=200, corr_slots=64, name="configs[4]: synthetic 1280x720, buffer=200")}
WL = WORKLOADS["cfg2"]


def set_workload(name):
    global WL, W_IMG, H_IMG
    WL = WORKLOADS[name]
    W_IMG, H_IMG = WL["w"], WL["h"]


def peaks():
    # NVIDIA's H100 SXM data sheet (700 W part): dense BF16 989 TFLOP/s, HBM3 3.35 TB/s -- data-sheet figures, not measured
    p = {"hbm_gbs": 3350.0, "bf16_tflops": 989.0, "_src": "H100 SXM data sheet"}
    f = os.path.join(ROOT, "MEASURED_PEAKS.json")
    if os.path.exists(f):
        p.update(json.load(open(f)))
        p["_src"] = "measured"
    return p


class ClockSampler:
    """nvidia-smi clocks/throttle reasons sampled DURING the timed region"""
    Q = "clocks.sm,clocks.max.sm,clocks_event_reasons.hw_slowdown,clocks_event_reasons.hw_thermal_slowdown," \
        "clocks_event_reasons.sw_thermal_slowdown,clocks_event_reasons.sw_power_cap"

    def __init__(self, index=0):
        self.rows, self.proc, self.index = [], None, index

    def start(self):
        try:
            self.proc = subprocess.Popen(["nvidia-smi", f"--query-gpu={self.Q}", "--format=csv,noheader,nounits",
                                          "-i", str(self.index), "-lms", "100"], stdout=subprocess.PIPE, text=True)
            self.t = threading.Thread(target=self._read, daemon=True)
            self.t.start()
        except Exception:
            self.proc = None

    def _read(self):
        for line in self.proc.stdout:
            self.rows.append([c.strip() for c in line.split(",")])

    def stop(self):
        if self.proc is None:
            return {"sm_mhz": None, "sm_max_mhz": None, "reasons": ["nvidia-smi unavailable"]}
        self.proc.terminate()
        try:
            self.proc.wait(timeout=2)
        except Exception:
            pass
        sm = [float(r[0]) for r in self.rows if r and r[0].replace(".", "").isdigit()]
        mx = [float(r[1]) for r in self.rows if len(r) > 1 and r[1].replace(".", "").isdigit()]
        names = ["hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown", "sw_power_cap"]
        reasons = sorted({names[i] for r in self.rows if len(r) >= 6 for i in range(4) if r[2 + i].lower().startswith("active")})
        return {"sm_mhz": float(np.median(sm)) if sm else None, "sm_max_mhz": max(mx) if mx else None,
                "reasons": reasons, "samples": len(sm)}


# ------------------------------------------------------------------------------------------ ours
def make_args(buffer):
    w = os.path.join(ROOT, "oracle", "_ref", "droid.pth")
    return types.SimpleNamespace(buffer=buffer, stereo=False, multi_gpu=False, eval=False, mask_type="ours",
                                 weights=w if os.path.exists(w) else None, corr_slots=WL["corr_slots"])


class SlamNerfJob:
    """single-process (N==1) or rank-local part of the job"""

    def __init__(self, rank, world, nerf_iters, buffer=100):
        import torch
        from nerf_slam_b200.synthetic import SyntheticRoom
        self.torch = torch
        self.rank, self.world, self.nerf_iters = rank, world, nerf_iters
        self.dev = torch.device("cuda", torch.cuda.current_device())
        self.is_slam = rank == 0
        self.is_nerf = (world == 1) or rank > 0
        self.room = SyntheticRoom(W_IMG, H_IMG, 100000, seed=0, step=STREAM_STEP)
        args = make_args(buffer)
        self.args = args
        self.fe = None
        self.nf = None
        self.k = 0
        self.h2d = self.d2h = 0
        self.launches = 0
        if self.is_slam:
            from nerf_slam_b200.frontend import RaftVisualFrontend
            self.fe = RaftVisualFrontend(np.linalg.inv(self.room.packet(0)["poses"][0]), np.eye(4), args, self.dev)
        if self.is_nerf:
            from nerf_slam_b200.nerf_fusion import NerfFusion
            self.nf = NerfFusion("nerf", args, self.dev)
            self.nerf_stream = torch.cuda.Stream(priority=0) if world == 1 else torch.cuda.current_stream()
            if world == 1 and "NSLAM_NERF_SMS" not in os.environ:
                # sharing the GPU with SLAM: the persistent NeRF kernels stay on about half of the SMs.  Unbounded, the
                # latency-critical SLAM kernels wait for NeRF CTAs to retire (persistent CTAs are not pre-empted); too
                # small a share stretches every NeRF kernel and with it the time both streams fight for the rest of the GPU.
                self.nf.ngp.num_sms = min(self.nf.ngp.num_sms, NERF_SM_BUDGET_SHARED)
        # SLAM is the latency-critical chain (host decisions wait on it): its kernels run on a HIGH-priority
        # stream so that NeRF training on the same GPU only fills the gaps
        self.slam_stream = torch.cuda.Stream(priority=-1) if (self.is_slam and world == 1) else torch.cuda.current_stream()
        self._res_ring = [torch.zeros(7).pin_memory() for _ in range(4)]
        self._res_events = [torch.cuda.Event() for _ in range(4)]
        self.handoff = None
        self.trainer = None
        if world > 1:
            import torch.distributed as dist
            from nerf_slam_b200 import dist as nd
            self.handoff = nd.Handoff(self.dev, 16, H_IMG, W_IMG)
            nerf_group = dist.new_group(list(range(1, world)))
            if self.is_nerf:
                nw = world - 1
                if nw > 1:
                    self.nf.ngp.grad_hook = lambda tb: nd.allreduce_grads(tb, nerf_group, nw)
                self.nf.ngp.seed = 1337 + 7919 * rank     # disjoint ray batches per trainer
                self.trainer = nd.TrainerLoop(self.handoff, self.nf, self._ingest, nerf_group, nw, device=self.dev)

    # frames -------------------------------------------------------------------------------
    def make_frames(self, n, on_device):
        """pre-render n frames (untimed). host: pinned uint8; device: uint8 CUDA tensors"""
        torch = self.torch
        out = []
        for _ in range(n):
            p = self.room.packet(self.k)
            self.k += 1
            img = torch.from_numpy(p["images"])
            p["images"] = img.to(self.dev) if on_device else img.pin_memory()
            p["depths"] = [None]                     # gt depth is not an input of the monocular path
            p["is_last_frame"] = False
            out.append(p)
        return out

    # one step -----------------------------------------------------------------------------
    def step(self, packet, e2e):
        torch = self.torch
        result = None
        if self.is_slam:
            if e2e:
                self.h2d += packet["images"].numel()
            with torch.cuda.stream(self.slam_stream):
                _, _, viz = self.fe.forward(packet)
                if self.world == 1:
                    if viz is not None and "cam0_poses" in viz:
                        ev = torch.cuda.Event(); ev.record()
                        with torch.cuda.stream(self.nerf_stream):
                            self.nerf_stream.wait_event(ev)
                            self.nf.process_slam([None, viz])
                else:
                    self._send(viz)
                if e2e:
                    # D2H of the step's result (latest keyframe pose): asynchronous copy into a pinned ring, consumed
                    # one step later -> the host never stalls on it; `drain_results` waits for the last ones before
                    # the timed region ends
                    slot = self.k % len(self._res_ring)
                    self._res_ring[slot].copy_(self.fe.cam0_T_world[max(self.fe.kf_idx - 1, 0)], non_blocking=True)
                    self._res_events[slot].record()
                    result = slot
                    self.d2h += 7 * 4
        if self.is_nerf and self.world == 1:
            with torch.cuda.stream(self.nerf_stream):
                for _ in range(self.nerf_iters):
                    self.nf.fit_volume_once()
            if e2e:
                self.d2h += 4
        return result

    def _send(self, viz):
        """rank 0: asynchronous hand-off of the dirty keyframes of this tick (nothing is sent on other frames)"""
        if viz is None or "cam0_poses" not in viz:
            return
        self.handoff.send(viz["viz_idx"], viz["cam0_poses"], viz["cam0_images"], viz["cam0_idepths_up"], viz["cam0_depths_cov_up"])

    def _ingest(self, idx, tq, img, idep, cov):
        intr = self.room.calib.camera_model.numpy()
        self.nf.ngp.nerf.training.update_training_images_device(idx.tolist(), None, img, idep, cov, intr[:2], intr[2:],
                                                                cam_T_world=tq)

    def drain_results(self):
        """all asynchronous result read-backs of the e2e arm have landed on the host"""
        for ev in self._res_events:
            ev.synchronize()
        return [r.clone() for r in self._res_ring]

    def sync(self):
        self.torch.cuda.synchronize()


def run_ours(a):
    # NCCL's version banner / debug lines go to a file, not to stdout (rank 0 prints exactly ONE JSON line)
    os.environ.setdefault("NCCL_DEBUG_FILE", "/tmp/nslam_nccl_%h_%p.log")
    # ... and whatever a library still writes to fd 1 (NCCL's version banner does) is diverted to stderr until
    # the result line is printed
    sys.stdout.flush()
    _saved_stdout = os.dup(1)
    os.dup2(2, 1)
    import torch
    rank = int(os.environ.get("RANK", 0)); world = int(os.environ.get("WORLD_SIZE", 1))
    local = int(os.environ.get("LOCAL_RANK", 0))
    torch.cuda.set_device(local)
    if world > 1:
        import torch.distributed as dist
        import datetime
        dist.init_process_group("nccl", device_id=torch.device("cuda", local), timeout=datetime.timedelta(minutes=30))
    assert world == a.gpus, f"--gpus {a.gpus} but WORLD_SIZE={world}"
    torch.set_grad_enabled(False)
    def barrier():
        torch.cuda.synchronize()
        if world > 1:
            import torch.distributed as dist
            dist.barrier()
        torch.cuda.synchronize()

    # keyframe buffer: the reference's default (100) holds ~500 frames of this stream (0.16 keyframes per frame);
    # longer runs get a proportionally larger buffer so that the timed region never reaches the buffer-full stop
    n_frames = a.steps + a.warmup + 40
    kf_buffer = WL["buffer"] if n_frames <= 4.6 * WL["buffer"] else int(24 + 0.2 * n_frames)

    def phase_end():
        """N > 1: rank 0 marks a phase boundary for the free-running trainers, then everybody meets at the barrier;
        trainers train (and ingest what arrives) until they see the marker"""
        if world > 1:
            from nerf_slam_b200 import dist as nd
            if job_ref[0].is_slam:
                nd.send_sync(job_ref[0].handoff)
            else:
                job_ref[0].trainer.run_until_sync()
        barrier()

    job_ref = [None]

    def new_primed_job():
        """fresh SLAM+NeRF state, primed (untimed) until SLAM is initialised and in steady state"""
        job = SlamNerfJob(rank, world, a.nerf_iters, buffer=kf_buffer)
        job_ref[0] = job
        primed = 0
        while job.is_slam:
            for p in job.make_frames(8, on_device=True):
                job.step(p, e2e=False)
                primed += 1
            if (job.fe.is_initialized and job.fe.kf_idx >= 12) or primed >= 400:
                break
        phase_end()
        return job, primed

    job, primed = new_primed_job()

    def timed(frames, e2e):
        if job.is_slam:
            for p in frames[:a.warmup]:
                job.step(p, e2e)
        phase_end()
        kf0 = job.fe.kf_idx if job.is_slam else 0
        up0 = job.fe.stats["updates"] if job.is_slam else 0
        it0 = job.nf.total_iters if job.is_nerf else 0
        e0 = torch.cuda.Event(enable_timing=True); e1 = torch.cuda.Event(enable_timing=True)
        prof = os.environ.get("NSLAM_CUDA_PROFILER") == "1" and not e2e
        if prof:
            torch.cuda.profiler.start()          # ncu --profile-from-start off captures only the timed region
        t0 = time.perf_counter()
        e0.record()
        if job.is_slam:
            for p in frames[a.warmup:]:
                job.step(p, e2e)
            if e2e:
                job.drain_results()
            if world == 1:
                torch.cuda.current_stream().wait_stream(job.nerf_stream)
                torch.cuda.current_stream().wait_stream(job.slam_stream)
            e1.record()
        # rank 0's device time ends here (e1); the trainers' ends when they have seen the phase marker — recorded after
        # the marker so that max-over-ranks covers hand-off completion on the receiving side too
        if world > 1 and job.is_slam:
            from nerf_slam_b200 import dist as nd
            nd.send_sync(job.handoff)
        elif world > 1:
            job.trainer.run_until_sync()
            e1.record()
        barrier()
        if prof:
            torch.cuda.profiler.stop()
        wall = time.perf_counter() - t0
        ms = e0.elapsed_time(e1)
        t = torch.tensor([ms], device=job.dev)
        n_it = torch.tensor([(job.nf.total_iters - it0) if job.is_nerf else 0], device=job.dev, dtype=torch.float32)
        n_it_max = n_it.clone()
        if world > 1:
            import torch.distributed as dist
            dist.all_reduce(t, op=dist.ReduceOp.MAX)
            dist.all_reduce(n_it, op=dist.ReduceOp.SUM)          # NeRF iterations of all trainer ranks
            dist.all_reduce(n_it_max, op=dist.ReduceOp.MAX)      # optimiser steps of the (data-parallel) model
        stats = dict(kf=(job.fe.kf_idx - kf0) if job.is_slam else 0, updates=(job.fe.stats["updates"] - up0) if job.is_slam else 0,
                     nerf_iters=int(n_it.item()), nerf_steps=int(n_it_max.item()), wall_s=wall)
        return float(t.item()), stats

    clocks = ClockSampler(local)
    dev_frames = job.make_frames(a.warmup + a.steps, on_device=True) if job.is_slam else []
    if rank == 0:
        clocks.start()
    ms_dev, st_dev = timed(dev_frames, e2e=False)
    clk = clocks.stop() if rank == 0 else None
    if a.dump_outputs and rank == 0:
        dump_outputs(job, a.dump_outputs)
    # the e2e arm starts from a fresh, re-primed state so that both arms see the same keyframe budget (buffer=100)
    job_ref[0] = None
    del dev_frames, job
    torch.cuda.empty_cache()
    job, _ = new_primed_job()
    host_frames = job.make_frames(a.warmup + a.steps, on_device=False) if job.is_slam else []
    job.h2d = job.d2h = 0
    ms_e2e, st_e2e = timed(host_frames, e2e=True)

    if world > 1:
        # everything below is rank 0's single-GPU post-processing: leave the process group cleanly first
        import torch.distributed as dist
        if job.is_slam:
            job.handoff.flush()
        barrier()
        dist.destroy_process_group()
    if rank != 0:
        return
    pk = peaks()
    fps = a.steps / (ms_dev / 1e3)
    fps_e2e = a.steps / (ms_e2e / 1e3)
    line = {
        "metric": "SLAM+NeRF frames/sec on 640x480 synthetic stream", "value": round(fps, 2), "unit": "frames/s",
        "n_gpus": world, "steps": a.steps, "warmup": a.warmup, "ms_per_step": round(ms_dev / a.steps, 3),
        "higher_is_better": True, "scaling": "strong", "vs_baseline": None, "dtype": "f16 operands + f32 accumulate (encoders, update operator, correlation, NeRF MLP) / f32 (BA, losses, Adam) / f64 (BA solve)",
        "data": "synthetic (procedural box room, seeded)",
        "config": {"workload": f"{WL['name']}, buffer={kf_buffer}, --slam --fusion=nerf",
                   "weights": "droid.pth" if job.args.weights else "random-init (seeded)", "nerf_iters_per_frame": a.nerf_iters,
                   "nerf_samples_per_iter": 1 << 18, "primed_frames": primed, "keyframes_in_timed_region": st_dev["kf"],
                   "update_calls_in_timed_region": st_dev["updates"], "nerf_iters_in_timed_region": st_dev["nerf_iters"],
                   "nerf_optimizer_steps_in_timed_region": st_dev["nerf_steps"],
                   "nerf_iters_per_s": round(st_dev["nerf_iters"] / (ms_dev / 1e3), 1),
                   "nerf_schedule": f"{a.nerf_iters} iterations per input frame on the SLAM GPU's second stream" if world == 1 else
                                    "free-running trainers (fit whenever no keyframe message is pending, fusion_module.py:30-33)",
                   "parallelism": "1 GPU: SLAM + NeRF on two streams" if world == 1 else f"rank0 SLAM, {world - 1} NeRF trainer rank(s) data-parallel over rays, asynchronous NCCL keyframe broadcast",
                   "l2": "inputs change every step and the working set exceeds L2; no explicit flush"},
        "e2e": {"value": round(fps_e2e, 2), "unit": "frames/s", "h2d_bytes_per_step": int(job.h2d / max(a.steps + a.warmup, 1)),
                "d2h_bytes_per_step": int(job.d2h / max(a.steps + a.warmup, 1)), "keyframes": st_e2e["kf"]},
        "clocks": clk,
    }
    st_dev["frames"] = a.steps
    shares, counts = kernel_shares(job, st_dev)
    entries = roofline_entries(job, pk)
    key, roof = pick_roofline(shares, entries)
    line["roofline"] = roof
    line["roofline_others"] = [v for k, v in entries.items() if k != key]
    line["kernel_shares"] = shares
    line["gpu_launches"] = counts["total"]
    line["gpu_launches_detail"] = counts
    if a.workload == "cfg4":
        # configs[3]: the global-BA pass (backend(): proximity graph over the whole window, update_lowmem on the alt-corr
        # path, window-wide BA) over the keyframes this run accumulated — timed on its own, not part of frames/s
        fe = job.fe
        with torch.cuda.stream(job.slam_stream):
            g0 = torch.cuda.Event(enable_timing=True); g1 = torch.cuda.Event(enable_timing=True)
            n_kf = fe.kf_idx
            g0.record(); fe.backend(steps=7); g1.record()
        torch.cuda.synchronize()
        line["global_ba"] = {"keyframes": int(n_kf), "max_factors": int(fe.max_factors), "steps": 7, "ms": round(g0.elapsed_time(g1), 2),
                             "ba_failures": fe.ba_failures(wait=True)}
    line["cpu_baseline"] = cpu_baseline_sample() if a.workload == "cfg2" else None
    sys.stdout.flush()
    os.dup2(_saved_stdout, 1)
    print(json.dumps(line), flush=True)


def dump_outputs(job, out_dir):
    """What the timed (device-resident) arm computed by its last step, as float32 .npy files in `out_dir`: the keyframe
    poses and inverse depths a SLAM caller receives, the last keyframe's full-resolution inverse depth, and the NeRF
    model (MLP weights and a fixed, seeded sample of the hash-grid parameters).  The stream and all seeds are fixed, so
    two builds run with the same arguments can be compared file by file; one build writes the same files on every
    run.  About 10 MB at the default workload."""
    import torch
    torch.cuda.synchronize()
    os.makedirs(out_dir, exist_ok=True)
    arrays = {}
    if job.is_slam:
        fe = job.fe
        k = int(fe.kf_idx)
        arrays["slam_keyframe_poses"] = fe.cam0_T_world[:k]
        arrays["slam_keyframe_idepths"] = fe.cam0_idepths[:k]
        arrays["slam_keyframe_idepths_cov"] = fe.cam0_idepths_cov[:k]
        arrays["slam_last_keyframe_idepth_up"] = fe.cam0_idepths_up[max(k - 1, 0)]
    if job.is_nerf:
        ngp = job.nf.ngp
        arrays["nerf_mlp_weights"] = ngp.mlp
        g = torch.Generator().manual_seed(0)
        n = ngp.grid_master.numel()
        idx = torch.randint(0, n, (min(n, 1 << 20),), generator=g).to(ngp.grid_master.device)
        arrays["nerf_grid_sample"] = ngp.grid_master[idx]
    for name, t in arrays.items():
        np.save(os.path.join(out_dir, name + ".npy"), t.detach().float().cpu().numpy())


def _time_kernel(torch, fn, dev, iters=8, skip=3):
    """CUDA-event timing on the launching (current) stream of ONE launch at a time, L2 flushed before each (a write
    of 256 MB > the 50 MB L2), device idle before and after: the isolated case -> compare with the BURST peaks"""
    flush = torch.empty(64 * 1024 * 1024, device=dev)
    ts = []
    for i in range(iters):
        flush.zero_()
        e0 = torch.cuda.Event(enable_timing=True); e1 = torch.cuda.Event(enable_timing=True)
        e0.record(); fn(); e1.record(); torch.cuda.synchronize()
        if i >= skip:
            ts.append(e0.elapsed_time(e1))
    return float(np.mean(ts))


def kernel_shares(job, st):
    """GPU-time share of every kernel in the timed region: CUPTI durations of one update(), one frame front and one NeRF
    iteration (own and library kernels alike), weighted by how often the timed region ran each.  Also returns the launch
    counts of OUR kernels (namespaces nslam:: / ngp::) for `gpu_launches`."""
    import torch
    from torch.profiler import profile, ProfilerActivity
    fe = job.fe

    def prof(fn):
        fn(); torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as pr:
            fn()
            torch.cuda.synchronize()
        t, own, n_all = {}, 0, 0
        for ev in pr.events():
            if ev.device_type == torch.autograd.DeviceType.CUDA and not ev.name.startswith("Mem"):
                n_all += 1
                own += ("nslam::" in ev.name or "ngp::" in ev.name)
                t[ev.name] = t.get(ev.name, 0.0) + ev.device_time_total
        return t, own, n_all
    img = job.make_frames(1, True)[0]
    x = img["images"].to(fe.device)[None].permute(0, 1, 4, 2, 3)
    with torch.cuda.stream(job.slam_stream):
        up = prof(lambda: fe.update(use_inactive=True))
        fr = prof(lambda: fe._frame_front(x))
    ne = ({}, 0, 0)
    if job.is_nerf:
        with torch.cuda.stream(job.nerf_stream):
            ne = prof(job.nf.fit_volume_once)
    tot = {}
    for (t, _, _), calls in ((up, st["updates"]), (fr, st["frames"]), (ne, st["nerf_iters"])):
        for k, v in t.items():
            tot[k] = tot.get(k, 0.0) + v * calls
    total_us = sum(tot.values()) or 1.0
    top = sorted(tot.items(), key=lambda kv: -kv[1])[:8]
    counts = {"total": int(up[1] * st["updates"] + fr[1] * st["frames"] + ne[1] * st["nerf_iters"]),
              "own_per_update_call": up[1], "all_per_update_call": up[2], "own_per_frame_front": fr[1],
              "all_per_frame_front": fr[2], "own_per_nerf_iter": ne[1], "all_per_nerf_iter": ne[2],
              "note": "own = kernels of libnslam_sm90a.so; the remainder are torch glue (index/copy/normalise) kernels; "
                      "per-keyframe extras (context encoder, correlation volumes of new edges) are not included in total"}
    shares = [{"kernel": k[:110], "share": round(v / total_us, 4)} for k, v in top]
    return shares, counts


def roofline_entries(job, pk):
    """isolated live timings (CUDA events, L2 flushed) of the kernels that carry the path, each against its bound;
    peaks: the BURST figures of MEASURED_PEAKS.json (a kernel timed alone)"""
    import ctypes
    import torch
    from nerf_slam_b200 import _lib, conv as nconv
    from nerf_slam_b200 import droid_backends as db
    fe, dev = job.fe, job.dev
    E, hw = int(fe.ii.shape[0]), fe.ht * fe.wd
    tf_peak, hbm_peak = pk["bf16_tflops"], pk["hbm_gbs"]
    src = pk["_src"] + " (burst figures: each kernel is timed alone, device idle around it)"
    out = {}

    def tensor_entry(key, name, flops, ms, extra=None):
        e = {"kernel": name, "bound": "tensor", "achieved": round(flops / ms / 1e9, 1), "peak": tf_peak, "unit": "TFLOP/s",
             "frac": round(flops / ms / 1e9 / tf_peak, 3), "launch_ms": round(ms, 4), "edges": E,
             "algorithmic_flops_per_launch": flops, "peak_source": src}
        e.update(extra or {})
        out[key] = e

    def hbm_entry(key, name, nbytes, ms, edges, extra=None):
        e = {"kernel": name, "bound": "hbm", "achieved": round(nbytes / ms / 1e6, 1), "peak": hbm_peak, "unit": "GB/s",
             "frac": round(nbytes / ms / 1e6 / hbm_peak, 3), "launch_ms": round(ms, 4), "edges": edges,
             "algorithmic_bytes_per_launch": nbytes, "peak_source": src}
        e.update(extra or {})
        out[key] = e
    op = fe.update_tc
    net = torch.randn(E, fe.ht, fe.wd, 128, device=dev).half(); inp = torch.randn_like(net); c2 = torch.randn_like(net)
    f2 = torch.randn(E, fe.ht, fe.wd, 64, device=dev).half()
    gzr = torch.zeros(E, 256, device=dev); z = torch.empty_like(net); rnet = torch.empty_like(net)
    wp, b = op.P["zr"]
    ms = _time_kernel(torch, lambda: nconv.conv_tc([net, inp, c2, f2], wp, b, E, fe.ht, fe.wd, 3, 1, 256, mode=1, gctx=gzr, net=net,
                                                   out0=z, out0_channels=128, out1=rnet, num_sms=op.num_sms), dev)
    tensor_entry("conv_zr", "conv_igemm_kernel<256,1> (A5: ConvGRU z|r gates, 3x3 448->256 + fused sigmoid / r*h epilogue)",
                 2.0 * E * hw * 9 * 448 * 256, ms)
    wq, bq = op.P["q"]
    gq = torch.zeros(E, 128, device=dev); hnew = torch.empty_like(net)
    ms = _time_kernel(torch, lambda: nconv.conv_tc([rnet, inp, c2, f2], wq, bq, E, fe.ht, fe.wd, 3, 1, 128, mode=2, gctx=gq, net=net,
                                                   zbuf=z, out0=hnew, out0_channels=128, num_sms=op.num_sms), dev)
    tensor_entry("conv_q", "conv_igemm_kernel<128,2> (A5: ConvGRU candidate state, 3x3 448->128 + fused tanh / state update)",
                 2.0 * E * hw * 9 * 448 * 128, ms)
    # the whole update operator (15 convolutions + glue kernels, one C call): FLOP-weighted aggregate of A5
    st = fe._static
    if st is not None and st.op_ctx is not None:
        ms = _time_kernel(torch, lambda: op.step(st.op_ctx), dev)
        tensor_entry("update_operator", "nslam_update_op_step (A5: all 15 wgmma implicit-GEMM convolutions + glue of UpdateModule.forward)",
                     2.0 * 2283008 * hw * E, ms, {"note": "2*2,283,008 MAC per edge-pixel (SURVEY.md §8a A5); includes the glue kernels' time"})
    # HBM-bound correlation kernels
    coords1, _ = fe.reproject(fe.ii, fe.jj)
    ms = _time_kernel(torch, lambda: fe.corr_pool.lookup(fe.slots_d, coords1, nhwc=True), dev)
    hbm_entry("corr_lookup", "corr_lookup_nhwc_kernel<half,3> (A3, 4 pyramid levels fused)",
              E * hw * (4 * 64 * 2 + 8 + nconv.CORR_PAD * 2), ms, E)
    lv = sum((fe.ht >> l) * (fe.wd >> l) for l in range(4))
    for Ev in (4, 16):
        fm = torch.randn(Ev + 1, fe.ht, fe.wd, 128, device=dev).half()
        ii32 = torch.arange(0, Ev, dtype=torch.int32, device=dev); jj32 = ii32 + 1
        ms = _time_kernel(torch, lambda: db.corr_volume_build(fm, ii32, jj32), dev)
        hbm_entry(f"corr_volume_E{Ev}", "corr_volume kernel (A2: all-pairs volume + 3 pooled levels in one pass)",
                  Ev * (2 * 128 * hw * 2 + hw * lv * 2), ms, Ev)
        del fm
    # the reference composite the volume kernel replaces: torch.matmul (cuBLAS) + 3x avg_pool2d (corr.py:23-38,63-72)
    Ev = 16
    f1 = torch.randn(Ev, 128, hw, device=dev).half(); f2_ = torch.randn(Ev, 128, hw, device=dev).half()

    def ref_volume():
        c = torch.matmul((f1 / 4.0).transpose(1, 2), f2_ / 4.0).view(Ev * hw, 1, fe.ht, fe.wd)
        for _ in range(3):
            c = torch.nn.functional.avg_pool2d(c, 2, stride=2)
    ms = _time_kernel(torch, ref_volume, dev)
    out["corr_volume_E16"]["library_composite_ms"] = round(ms, 4)
    # the volume kernel only WRITES (features are L2-resident): the write-only ceiling of this GPU, measured with a plain
    # fill of the same size, next to the copy figure `peak` is quoted against
    nb = out["corr_volume_E16"]["algorithmic_bytes_per_launch"]
    fillbuf = torch.empty(nb, dtype=torch.uint8, device=dev)
    ms_fill = _time_kernel(torch, lambda: fillbuf.zero_(), dev)
    out["corr_volume_E16"]["write_only_fill_gbs"] = round(nb / ms_fill / 1e6, 1)
    out["corr_volume_E16"]["frac_of_write_only_fill"] = round(out["corr_volume_E16"]["achieved"] / (nb / ms_fill / 1e6), 3)
    del fillbuf
    out["corr_volume_E16"]["library_composite"] = "torch.matmul fp16 + 3x avg_pool2d at the same 16 edges (what CorrBlock.__init__ runs)"
    del f1, f2_
    # NeRF (B3): the tensor-core MLP backward = largest single kernel of the trainer
    if job.is_nerf:
        tb = job.nf.ngp
        lib = _lib.load()
        with torch.cuda.stream(job.nerf_stream):
            tb.train_step(); torch.cuda.synchronize()
        n = int(tb._bufs["counters"][0].item())
        bufs = tb._bufs
        with torch.cuda.stream(job.nerf_stream):
            def bwd():
                _lib.check(lib.nslam_ngp_backward_tc(ctypes.byref(tb.model), _lib.ptr(tb.packed), _lib.ptr(bufs["coords"]),
                                                     _lib.ptr(bufs["counters"]), _lib.ptr(bufs["dout"]), float(tb.loss_scale),
                                                     _lib.ptr(bufs["enc"]), _lib.ptr(bufs["denc"]), tb.max_samples, tb.num_sms,
                                                     ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)), "backward_tc")
            ms = _time_kernel(torch, bwd, dev)
            ms_step = _time_kernel(torch, tb.train_step, dev)
        tensor_entry("ngp_backward", "ngp::backward_tc_kernel (+ grid scatter) (B3: MLP backward on wgmma, recompute + dW + dX)",
                     3.0 * 2 * 10240 * n, ms, {"samples": n, "num_sms": tb.num_sms, "edges": None,
                                               "note": "3 x forward MACs (recompute, dW, dX) x samples of one batch"})
        out["ngp_backward"]["train_step_ms"] = round(ms_step, 4)
    return out


def pick_roofline(shares, entries):
    """the `roofline` object = the entry of the kernel with the LARGEST GPU-time share of the timed region that has an
    isolated timing; the FLOP-weighted aggregate of the update operator and everything else go to roofline_others"""
    table = (("conv_igemm_kernel<256, 1", "conv_zr"), ("conv_igemm_kernel<128, 2", "conv_q"), ("backward_tc", "ngp_backward"),
             ("corr_lookup_nhwc", "corr_lookup"), ("corr_volume", "corr_volume_E4"))
    for s in shares:
        for needle, key in table:
            if needle in s["kernel"] and key in entries:
                e = dict(entries[key])
                e["share_of_gpu_time_in_timed_region"] = s["share"]
                return key, e
    return "conv_zr", dict(entries["conv_zr"])


def cpu_baseline_sample(max_seconds=40.0):
    """reference's CPU-only PyTorch path (oracle/cpu_path.py) on this box's host cores: steady-state cycles of the same
    workload, timed directly (one untimed warm-up cycle first: thread pools, oneDNN primitives)"""
    from oracle import cpu_path as cp
    w = os.path.join(ROOT, "oracle", "_ref", "droid.pth")
    path = cp.CpuPath(w if os.path.exists(w) else None)
    path.frame_front(); path.candidate_setup(); path.update()          # warm-up (untimed)
    secs, parts_sum, n = 0.0, None, 0
    t0 = time.perf_counter()
    while n == 0 or (time.perf_counter() - t0) + secs / max(n, 1) < max_seconds:
        t, parts = cp.steady_state_cycle(path)
        secs += t; n += 1
        parts_sum = parts if parts_sum is None else {k: parts_sum[k] + v for k, v in parts.items()}
    per = secs / n
    return {"value": round(cp.CYCLE["frames"] / per, 4), "unit": "frames/s", "cores": cp.host_threads(), "kind": "port",
            "sample": cp.sample_description(per, {k: v / n for k, v in parts_sum.items()}, n), "cycles": n}


# ------------------------------------------------------------------------------------------ reference arms
def _ref_line(a, impl, value, steps, extra):
    line = {"impl": impl, "metric": "SLAM+NeRF frames/sec on 640x480 synthetic stream", "value": round(value, 4),
            "unit": "frames/s", "n_gpus": a.gpus, "steps": steps, "warmup": a.warmup,
            "ms_per_step": round(1e3 / max(value, 1e-9), 2), "higher_is_better": True, "scaling": "strong", "vs_baseline": None,
            "data": "synthetic (procedural box room, seeded)",
            "e2e": {"value": round(value, 4), "unit": "frames/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0}}
    line.update(extra)
    return line


def run_reference(a):
    """--impl reference: the reference's CPU-only PyTorch path on this box's host cores (rank 0 only).  A step = one
    frame of the steady-state cycle of oracle/cpu_path.py; cycles are timed directly until --steps frames or ~150 s."""
    if int(os.environ.get("RANK", 0)) != 0:
        return
    from oracle import cpu_path as cp
    w = os.path.join(ROOT, "oracle", "_ref", "droid.pth")
    path = cp.CpuPath(w if os.path.exists(w) else None)
    for _ in range(1 if a.warmup > 0 else 0):
        path.frame_front(); path.candidate_setup(); path.update()
    secs, parts_sum, n = 0.0, None, 0
    t0 = time.perf_counter()
    want = max(1, -(-a.steps // cp.CYCLE["frames"]))
    while n < want and (n == 0 or (time.perf_counter() - t0) + secs / n < 150.0):
        t, parts = cp.steady_state_cycle(path)
        secs += t; n += 1
        parts_sum = parts if parts_sum is None else {k: parts_sum[k] + v for k, v in parts.items()}
    per = secs / n
    v = cp.CYCLE["frames"] / per
    base = {"value": round(v, 4), "unit": "frames/s", "cores": cp.host_threads(), "kind": "port",
            "sample": cp.sample_description(per, {k: x / n for k, x in parts_sum.items()}, n)}
    print(json.dumps(_ref_line(a, "reference", v, n * cp.CYCLE["frames"], {
        "dtype": "f32 (networks, correlation) / f64 (BA)",
        "config": {"workload": "configs[1]: Replica-office0-shaped synthetic 640x480, buffer=100, --slam --fusion=nerf",
                   "note": "reference's CPU-only PyTorch path on a bounded sample of this workload (steady-state cycles), see cpu_baseline.sample"},
        "cpu_baseline": base})), flush=True)


def run_reference_cuda(a):
    """--impl reference-cuda: the reference's OWN CUDA kernels (oracle/_ref, compiled from /root/reference/src) + library
    PyTorch in the reference's sequencing (oracle/ref_cuda_frontend.py) on the SAME stream, same priming, same timing
    rules as the product arm; SLAM only (the reference's NeRF is the absent instant-ngp fork).  One GPU."""
    if int(os.environ.get("RANK", 0)) != 0:
        return
    sys.stdout.flush()
    saved = os.dup(1); os.dup2(2, 1)
    import torch
    from nerf_slam_b200.synthetic import SyntheticRoom
    from oracle.ref_cuda_frontend import RefCudaFrontend
    torch.cuda.set_device(0)
    torch.set_grad_enabled(False)
    dev = torch.device("cuda", 0)
    room = SyntheticRoom(W_IMG, H_IMG, 100000, seed=0, step=STREAM_STEP)
    n_frames = a.steps + a.warmup + 40
    fe = RefCudaFrontend(np.linalg.inv(room.packet(0)["poses"][0]), np.eye(4), make_args(100 if n_frames <= 460 else int(24 + 0.2 * n_frames)), dev)
    k = 0

    def frames(n):
        nonlocal k
        out = []
        for _ in range(n):
            p = room.packet(k); k += 1
            p["images"] = torch.from_numpy(p["images"]).to(dev); p["depths"] = [None]; p["is_last_frame"] = False
            out.append(p)
        return out
    primed = 0
    while not (fe.is_initialized and fe.kf_idx >= 12) and primed < 400:
        for p in frames(8):
            fe.forward(p); primed += 1
    torch.cuda.synchronize()
    fr = frames(a.warmup + a.steps)
    for p in fr[:a.warmup]:
        fe.forward(p)
    torch.cuda.synchronize()
    kf0, up0 = fe.kf_idx, fe.stats["updates"]
    clocks = ClockSampler(0); clocks.start()
    e0 = torch.cuda.Event(enable_timing=True); e1 = torch.cuda.Event(enable_timing=True)
    e0.record()
    for p in fr[a.warmup:]:
        fe.forward(p)
    e1.record(); torch.cuda.synchronize()
    clk = clocks.stop()
    ms = e0.elapsed_time(e1)
    v = a.steps / (ms / 1e3)
    sys.stdout.flush(); os.dup2(saved, 1)
    print(json.dumps(_ref_line(a, "reference-cuda", v, a.steps, {
        "dtype": "f16 autocast (networks, correlation) / f32 (kernels) / f64 (host solve)",
        "config": {"workload": "configs[1]: Replica-office0-shaped synthetic 640x480, --slam (NeRF not included: instant-ngp fork absent)",
                   "implementation": "reference CUDA kernels from oracle/_ref + library PyTorch in the reference's sequencing; gtsam / lietorch "
                                     "replaced by faster stand-ins (oracle/ref_cuda_frontend.py)",
                   "primed_frames": primed, "keyframes_in_timed_region": fe.kf_idx - kf0,
                   "update_calls_in_timed_region": fe.stats["updates"] - up0},
        "clocks": clk})), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=192)
    ap.add_argument("--warmup", type=int, default=8)
    ap.add_argument("--impl", default="ours", choices=["ours", "reference", "reference-cuda"])
    ap.add_argument("--nerf-iters", type=int, default=2)
    ap.add_argument("--workload", default="cfg2", choices=sorted(WORKLOADS))
    ap.add_argument("--dump-outputs", metavar="DIR", default=None,
                    help="write what the timed path computed in its last step as DIR/<name>.npy (float32)")
    a = ap.parse_args()
    set_workload(a.workload)
    if a.impl == "reference":
        run_reference(a)
    elif a.impl == "reference-cuda":
        run_reference_cuda(a)
    else:
        run_ours(a)


if __name__ == "__main__":
    main()
