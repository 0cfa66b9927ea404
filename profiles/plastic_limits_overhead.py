"""Cost of the plastic yield limits (MPMSimulator.set_plastic_limits) bound at their defaults, against the table, timed with CUDA events in
alternation (--pairs runs of each setting, so that all see the same machine state), on 1M ICECREAM particles at C2's positions (bench.py's
workload with the material changed) on 64^3: ICECREAM on bench.py's 128^3 is beyond the fixed time step (dt c / dx > 1), its state turns NaN
within the first steps and the timing would be of NaN arithmetic:
  fwd  forward-only steps (fused k_fwd path, CUDA graphs): substeps per second
  fb   forward + backward of --steps steps with the T = 50 ring, sort every 4 steps and param_grad on
Settings: the table (k_fwd<0>, k_particle_grad<0, *>), and the limits at their defaults (mu, lam and mass per slot gathered from the rows:
k_fwd<4>, k_particle_grad<4, *>), each on a simulator of its own with its fields bound once; the forward runs start one untimed step after
set_state.  Prints one JSON line with median and min-max of each, the card and its power limit.   python profiles/plastic_limits_overhead.py"""
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
from fluidlab_b200 import MPMSimulator, macros as M  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument('--steps', type=int, default=10)
ap.add_argument('--fwd-steps', type=int, default=50)
ap.add_argument('--pairs', type=int, default=5)
args = ap.parse_args()
assert torch.cuda.is_available(), 'needs a CUDA device'
N = bench.N_PARTICLES
sys.path.insert(0, os.path.join(ROOT, 'tests'))
from conftest import make_particles  # noqa: E402
xw = bench.workload_particles(N)['x']


def make(limits):
    P = make_particles(xw, M.ICECREAM, 64)
    s = MPMSimulator(dim=3, quality=1.0, gravity=bench.GRAVITY, horizon=400, max_substeps_local=50, max_substeps_global=10 ** 7,
                     ckpt_dest='gpu', sort_every=4)
    s.build(None, None, [], P)
    s.fuse_g2p2g = True
    if limits:
        s.set_plastic_limits()
    return s, s.get_state()


def fwd(s, init):
    s.disable_grad(); s.set_state(0, init)
    s.step(None)   # untimed: the first step after set_state gathers the fields into its slot order
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(args.fwd_steps):
        s.step(None)
    b.record(); torch.cuda.synchronize()
    return args.fwd_steps * s.n_substeps / (a.elapsed_time(b) * 1e-3)


def fwd_bwd(s, init, tgt, mask):
    s.param_grad = True
    s.set_state(0, init); s.enable_grad()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(args.steps):
        s.step(None)
    s.reset_grad()
    s.add_x_grad_chamfer(tgt, mask, 1.0)
    for _ in range(args.steps):
        s.step_grad(None)
    b.record(); torch.cuda.synchronize()
    return a.elapsed_time(b)


stat = lambda a: dict(median=float(np.median(a)), min=float(min(a)), max=float(max(a)))
sims = {lim: make(lim) for lim in (False, True)}
dev = sims[False][0].device
tgt = torch.zeros((N, 3), dtype=torch.float32, device=dev) + 0.5
mask = sims[False][0].material_row_mask(M.ICECREAM)
for lim in (False, True):   # warm-up of every kernel set and of the graphs
    fwd(*sims[lim]); fwd_bwd(*sims[lim], tgt, mask)
res = {k: {lim: [] for lim in (False, True)} for k in ('fwd', 'fb')}
for _ in range(args.pairs):
    for lim in (False, True):
        res['fwd'][lim].append(fwd(*sims[lim]))
        res['fb'][lim].append(fwd_bwd(*sims[lim], tgt, mask))
g = sims[True][0].get_param_grad()
assert np.isfinite(g['theta_c']).all() and np.isfinite(g['theta_s']).all(), 'the ICECREAM run stays finite'
out = {}
for lim, name in ((False, 'table'), (True, 'limits')):
    out[f'icecream_fwd_substeps_per_s_{name}'] = stat(res['fwd'][lim])
    out[f'icecream_fwd_bwd_ms_{name}'] = stat(res['fb'][lim])
out['icecream_fwd_cost_ratio_limits_vs_table'] = float(np.median(res['fwd'][False]) / np.median(res['fwd'][True]))
out['icecream_fwd_bwd_cost_ratio_limits_vs_table'] = float(np.median(res['fb'][True]) / np.median(res['fb'][False]))
out['theta_grad_rows'] = [float(g['theta_c'][0]), float(g['theta_s'][0])]
gpu = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader', '-i', str(dev.index or 0)],
                     capture_output=True, text=True).stdout.strip()
print(json.dumps(dict(gpu=gpu, particles=N, steps=args.steps, fwd_steps=args.fwd_steps, pairs=args.pairs, **out)))
