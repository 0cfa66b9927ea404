"""Cost of a per-particle material field (MPMSimulator.set_material_field) against the material table alone: 1M ELASTIC particles in C2's box at
128^3 (bench.py's workload with the material changed, so that the table run also takes the general k_fwd and the comparison isolates the
field), with the field equal to the table.  Timed with CUDA events, the two settings in alternation (--pairs runs each), so that both see the
same machine state:
  fwd   forward-only steps (fused k_fwd path, CUDA graphs): substeps per second
  fb    forward + backward of --steps steps with the T = 50 ring, sort every 4 steps and param_grad on (chunk re-simulation included)
Prints one JSON line with median and min-max of each, the card and its power limit.   python profiles/material_field_overhead.py"""
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
P = make_particles(bench.workload_particles(N)['x'], M.ELASTIC, int(64 * bench.QUALITY))   # C2's positions, ELASTIC
sim = MPMSimulator(dim=3, quality=bench.QUALITY, gravity=bench.GRAVITY, horizon=400, max_substeps_local=50, max_substeps_global=10 ** 7, ckpt_dest='gpu', sort_every=4)
sim.build(None, None, [], P)
sim.fuse_g2p2g = True
init = sim.get_state()
mu, lam = np.asarray(P['mu']), np.asarray(P['lam'])
tgt = torch.zeros((N, 3), dtype=torch.float32, device=sim.device) + 0.5
mask = sim.material_row_mask(M.ELASTIC)


def use(field):
    if field:
        sim.set_material_field(mu, lam)
    else:
        sim.clear_material_field()


def fwd(field):
    use(field)
    sim.disable_grad(); sim.set_state(0, init)
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(args.fwd_steps):
        sim.step(None)
    b.record(); torch.cuda.synchronize()
    return args.fwd_steps * sim.n_substeps / (a.elapsed_time(b) * 1e-3)


def fwd_bwd(field):
    use(field)
    sim.param_grad = True
    sim.set_state(0, init); sim.enable_grad()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(args.steps):
        sim.step(None)
    sim.reset_grad()
    sim.add_x_grad_chamfer(tgt, mask, 1.0)
    for _ in range(args.steps):
        sim.step_grad(None)
    b.record(); torch.cuda.synchronize()
    return a.elapsed_time(b)


for field in (False, True):   # warm-up of both kernel sets and of the graphs
    fwd(field); fwd_bwd(field)
res = {k: {False: [], True: []} for k in ('fwd', 'fb')}
for _ in range(args.pairs):
    for field in (False, True):
        res['fwd'][field].append(fwd(field))
        res['fb'][field].append(fwd_bwd(field))
g = sim.get_param_grad()
stat = lambda a: dict(median=float(np.median(a)), min=float(min(a)), max=float(max(a)))
gpu = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader', '-i', str(sim.device.index or 0)],
                     capture_output=True, text=True).stdout.strip()
out = dict(gpu=gpu, particles=N, material='ELASTIC', fwd_substeps_per_s_table=stat(res['fwd'][False]), fwd_substeps_per_s_field=stat(res['fwd'][True]),
           fwd_bwd_ms_table=stat(res['fb'][False]), fwd_bwd_ms_field=stat(res['fb'][True]), steps=args.steps, pairs=args.pairs,
           fwd_cost_ratio=float(np.median(res['fwd'][False]) / np.median(res['fwd'][True])),
           fwd_bwd_cost_ratio=float(np.median(res['fb'][True]) / np.median(res['fb'][False])),
           mu_field_finite=bool(np.isfinite(g['mu_field']).all()), mu_row_vs_field_sum=[float(g['mu'][0]), float(g['mu_field'].sum())])
print(json.dumps(out))
