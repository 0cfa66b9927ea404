"""Cost of a per-particle density field (MPMSimulator.set_density_field), every field equal to the table, timed with CUDA events in alternation
(--pairs runs of each setting, so that all see the same machine state):
  elastic  1M ELASTIC particles at C2's positions on 128^3 (bench.py's workload with the material changed, so that the table run takes the
           general k_fwd too), settings table / mu, lam field / mu, lam + rho field:
             fwd  forward-only steps (fused k_fwd path, CUDA graphs): substeps per second
             fb   forward + backward of --steps steps with the T = 50 ring, sort every 4 steps and param_grad on
  water    C2 itself (all-liquid: the k_fwd<1> table path) against C2 with a rho field (the general kernels with mu, lam and mass per slot):
           forward substeps per second
  loss     per-call time of fmpm_loss_density(_grad) and fmpm_loss_momentum(_grad) on the elastic scene's frame, without and with the field
Every setting has a simulator of its own with its fields bound once, so no timed run pays a rebinding (a CUDA-graph recapture and a field
gather); the forward runs start one untimed step after set_state.  Prints one JSON line with median and min-max of each, the card and its power
limit.   python profiles/density_field_overhead.py"""
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
ap.add_argument('--loss-calls', type=int, default=50)
args = ap.parse_args()
assert torch.cuda.is_available(), 'needs a CUDA device'
N = bench.N_PARTICLES
sys.path.insert(0, os.path.join(ROOT, 'tests'))
from conftest import make_particles  # noqa: E402
xw = bench.workload_particles(N)['x']


def make(mat, setting):
    """setting 0: the table, 1: a (mu, lam) field, 2: a (mu, lam) field and a rho field, 3: a rho field alone; all equal to the rows"""
    P = make_particles(xw, mat, int(64 * bench.QUALITY))
    s = MPMSimulator(dim=3, quality=bench.QUALITY, gravity=bench.GRAVITY, horizon=400, max_substeps_local=50, max_substeps_global=10 ** 7,
                     ckpt_dest='gpu', sort_every=4)
    s.build(None, None, [], P)
    s.fuse_g2p2g = True
    if setting in (1, 2):
        s.set_material_field(P['mu'], P['lam'])
    if setting in (2, 3):
        s.set_density_field(P['rho'])
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


def loss_calls(s, init, bufs):
    """ms per call of the four loss entry points on frame 0 of the elastic scene"""
    s.set_state(0, init); s.enable_grad(); s.reset_grad()
    mass, fld, out, mask = bufs
    calls = dict(density=lambda: s.density_loss(mass, None, None, 1.0, 0.0, mask, out, f=0),
                 density_grad=lambda: s.add_x_grad_density(mass, None, None, 1.0, 0.0, mask, f=0),
                 momentum=lambda: s.momentum_loss(fld, None, None, 1.0, 0.0, 1.0, mask, out, f=0),
                 momentum_grad=lambda: s.add_grad_momentum(fld, None, None, 1.0, 0.0, 1.0, mask, f=0))
    res = {}
    for k, fn in calls.items():
        fn(); torch.cuda.synchronize()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(args.loss_calls):
            fn()
        b.record(); torch.cuda.synchronize()
        res[k] = a.elapsed_time(b) / args.loss_calls
    return res


stat = lambda a: dict(median=float(np.median(a)), min=float(min(a)), max=float(max(a)))
out = {}
# ---- elastic: table / field / field + rho (the loss calls: table / field + rho, whose losses read the rho field)
settings = (0, 1, 2)
sims = {st: make(M.ELASTIC, st) for st in settings}
dev = sims[0][0].device
tgt = torch.zeros((N, 3), dtype=torch.float32, device=dev) + 0.5
mask = sims[0][0].material_row_mask(M.ELASTIC)
G = sims[0][0].n_grid ** 3
bufs = (torch.zeros(G, dtype=torch.float32, device=dev), torch.zeros((G, 4), dtype=torch.float32, device=dev),
        torch.zeros(1, dtype=torch.float32, device=dev), mask)
for st in settings:   # warm-up of every kernel set and of the graphs
    s, ini = sims[st]
    fwd(s, ini); fwd_bwd(s, ini, tgt, mask); loss_calls(s, ini, bufs)
res = {k: {st: [] for st in settings} for k in ('fwd', 'fb')}
lres = {st: [] for st in (0, 2)}
for _ in range(args.pairs):
    for st in settings:
        s, ini = sims[st]
        res['fwd'][st].append(fwd(s, ini))
        res['fb'][st].append(fwd_bwd(s, ini, tgt, mask))
    for st in (0, 2):
        lres[st].append(loss_calls(*sims[st], bufs))
g = sims[2][0].get_param_grad()
names = {0: 'table', 1: 'field', 2: 'field_rho'}
for st in settings:
    out[f'elastic_fwd_substeps_per_s_{names[st]}'] = stat(res['fwd'][st])
    out[f'elastic_fwd_bwd_ms_{names[st]}'] = stat(res['fb'][st])
out['elastic_fwd_cost_ratio_field_rho_vs_table'] = float(np.median(res['fwd'][0]) / np.median(res['fwd'][2]))
out['elastic_fwd_cost_ratio_field_rho_vs_field'] = float(np.median(res['fwd'][1]) / np.median(res['fwd'][2]))
out['elastic_fwd_bwd_cost_ratio_field_rho_vs_table'] = float(np.median(res['fb'][2]) / np.median(res['fb'][0]))
out['elastic_fwd_bwd_cost_ratio_field_rho_vs_field'] = float(np.median(res['fb'][2]) / np.median(res['fb'][1]))
out['rho_row_vs_field_sum'] = [float(g['rho'][0]), float(g['rho_field'].sum())]
for k in ('density', 'density_grad', 'momentum', 'momentum_grad'):
    out[f'loss_ms_per_call_{k}_table'] = stat([r[k] for r in lres[0]])
    out[f'loss_ms_per_call_{k}_rho'] = stat([r[k] for r in lres[2]])
del sims, s, ini, bufs
torch.cuda.empty_cache()
# ---- water (C2): the all-liquid table path against a rho field
wsims = {st: make(M.WATER, st) for st in (0, 3)}
for st in (0, 3):
    fwd(*wsims[st])
wres = {0: [], 3: []}
for _ in range(args.pairs):
    for st in (0, 3):
        wres[st].append(fwd(*wsims[st]))
out['water_fwd_substeps_per_s_table'] = stat(wres[0])
out['water_fwd_substeps_per_s_rho'] = stat(wres[3])
out['water_fwd_cost_ratio_rho_vs_table'] = float(np.median(wres[0]) / np.median(wres[3]))
gpu = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader', '-i', str(dev.index or 0)],
                     capture_output=True, text=True).stdout.strip()
print(json.dumps(dict(gpu=gpu, particles=N, steps=args.steps, fwd_steps=args.fwd_steps, pairs=args.pairs, **out)))
