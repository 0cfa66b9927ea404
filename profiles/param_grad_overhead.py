"""Cost of MPMSimulator.param_grad (loss gradients with respect to the material rows and gravity) on the C2 workload of bench.py (1M water
particles, 128^3, the reference's T = 50 ring, sort every 4 steps, fused forward): the forward + backward pass of bench.py's `fwd_bwd` (10 steps,
chunk re-simulation included), timed with CUDA events with param_grad off and on in alternation, so that both see the same machine state.
Prints one JSON line with the card and its power limit.   python profiles/param_grad_overhead.py [--steps 10] [--pairs 5]"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402
import fluidlab_b200  # noqa: E402
from fluidlab_b200 import MPMSimulator  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument('--steps', type=int, default=10)
ap.add_argument('--pairs', type=int, default=5)
args = ap.parse_args()
assert torch.cuda.is_available(), 'needs a CUDA device'
N, nfb = bench.N_PARTICLES, args.steps
sim = MPMSimulator(dim=3, quality=bench.QUALITY, gravity=bench.GRAVITY, horizon=400, max_substeps_local=50, max_substeps_global=10 ** 7, ckpt_dest='gpu', sort_every=4)
sim.build(None, None, [], bench.workload_particles(N))
sim.fuse_g2p2g = True
init = sim.get_state()
tgt = torch.zeros((N, 3), dtype=torch.float32, device=sim.device) + 0.5
mask = sim.material_row_mask(fluidlab_b200.macros.WATER)


def fwd_bwd(pg):
    sim.param_grad = pg
    sim.set_state(0, init); sim.enable_grad()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(nfb):
        sim.step(None)
    sim.reset_grad()
    sim.add_x_grad_chamfer(tgt, mask, 1.0)
    for _ in range(nfb):
        sim.step_grad(None)
    b.record(); torch.cuda.synchronize()
    return a.elapsed_time(b)


fwd_bwd(False); fwd_bwd(True)   # warm-up of both kernel sets and of the graphs
runs = {False: [], True: []}
for _ in range(args.pairs):
    for pg in (False, True):
        runs[pg].append(fwd_bwd(pg))
g = sim.get_param_grad()
off, on = float(np.median(runs[False])), float(np.median(runs[True]))
gpu = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader', '-i', str(sim.device.index or 0)],
                     capture_output=True, text=True).stdout.strip()
print(json.dumps(dict(gpu=gpu, steps=nfb, substep_pairs_per_s_default=nfb * 10 / (off * 1e-3), substep_pairs_per_s_param_grad=nfb * 10 / (on * 1e-3),
                      overhead_ratio=on / off, runs_ms_default=runs[False], runs_ms_param_grad=runs[True],
                      spread_default=(max(runs[False]) - min(runs[False])) / off, spread_param_grad=(max(runs[True]) - min(runs[True])) / on,
                      dL_dg=[float(v) for v in g['gravity']], finite=bool(np.isfinite(g['gravity']).all()))))
