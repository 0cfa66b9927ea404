"""Cost of the correspondence-free momentum loss (MomentumMatchingLoss: fmpm_loss_momentum / fmpm_loss_momentum_grad) on the C2 workload of
bench.py (1M water particles, 128^3, the reference's T = 50 ring, sort every 4 steps, fused forward).

1. A TaichiEnv forward + backward pass of --steps steps with the loss evaluated and seeded at every step, timed with CUDA events, with the
   index-matched ShapeMatchingLoss, with DensityMatchingLoss (density and SDF terms) and with MomentumMatchingLoss (density, SDF and
   momentum terms), alternated run by run so that all see the same machine state: median (min - max) of --runs runs each.
2. The device time per call of both momentum entry points (CUDA events) and per launch of the momentum kernels, the density deposit and
   k_fwd (torch.profiler, CUDA activities) over --launches calls each, on a cell-sorted frame and on a frame in the particles' original order.
Prints one JSON line, with the card and its power limit read in the same run.
    python profiles/momentum_loss_overhead.py [--steps 10] [--runs 5] [--launches 200]"""
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
from fluidlab_b200 import TaichiEnv, ShapeMatchingLoss, DensityMatchingLoss, MomentumMatchingLoss, macros as M  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument('--steps', type=int, default=10)
ap.add_argument('--runs', type=int, default=5)
ap.add_argument('--launches', type=int, default=200)
args = ap.parse_args()
assert torch.cuda.is_available(), 'needs a CUDA device'
N, steps = bench.N_PARTICLES, args.steps
P = bench.workload_particles(N)
env = TaichiEnv(quality=bench.QUALITY, max_substeps_local=50, max_substeps_global=10 ** 7, gravity=bench.GRAVITY, horizon=steps, sort_every=4)
env.particle_bodies.get = lambda: P
env.build()
sim = env.simulator
sim.fuse_g2p2g = True
init = sim.get_state()
n = sim.n_grid
x0 = np.asarray(P['x'], np.float64)
m_p = float(np.float32(sim.p_vol) * np.float32(sim.get_material_table()['rho'][0]))
shape = ShapeMatchingLoss(M.WATER, max_loss_steps=steps, weights={'chamfer': 1.0}, temporal_range_type='all',
                          target=[(x0 + [0.01, -0.02, 0.0]).astype(np.float32)] * steps)
ax = np.arange(n) / n
X, Y, Z = np.meshgrid(ax, ax, ax, indexing='ij')
sdf = (np.sqrt((X - 0.5) ** 2 + (Y - 0.4) ** 2 + (Z - 0.5) ** 2) - 0.2).reshape(-1)
dens = DensityMatchingLoss(M.WATER, max_loss_steps=steps, weights={'density': 1.0 / m_p ** 2, 'sdf': 1.0 / m_p}, temporal_range_type='all',
                           target=DensityMatchingLoss.density_from_points(x0 + [0.02, -0.03, 0.0], m_p, n), target_sdf=sdf)
tp = 2 * np.pi
u_star = 0.3 * np.stack([np.cos(tp * x0[:, 1] * 2), np.sin(tp * x0[:, 2] * 2), np.cos(tp * x0[:, 0] * 3)], 1)
p_star, m_star = MomentumMatchingLoss.momentum_from_points(x0 + [0.02, -0.03, 0.0], u_star, m_p, n)
mom = MomentumMatchingLoss(M.WATER, max_loss_steps=steps, weights={'density': 1.0 / m_p ** 2, 'sdf': 1.0 / m_p, 'momentum': 1.0 / m_p ** 2},
                           temporal_range_type='all', target=m_star, target_sdf=sdf, target_momentum=p_star)
shape.build(sim); dens.build(sim); mom.build(sim)


def fwd_bwd(loss):
    env.loss = loss
    env.set_state(init, grad_enabled=True)
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(steps):
        env.step()
    env.get_final_loss()
    env.reset_grad(); env.get_final_loss_grad()
    for _ in range(steps):
        env.step_grad()
    b.record(); torch.cuda.synchronize()
    return a.elapsed_time(b)


losses = dict(shape=shape, density=dens, momentum=mom)
for k in losses:
    fwd_bwd(losses[k])   # warm-up of both losses and of the graphs
runs = {k: [] for k in losses}
for _ in range(args.runs):
    for k in losses:
        runs[k].append(fwd_bwd(losses[k]))
total = float(mom.step_loss.sum().item())

# per-call and per-kernel device times on the frame the backward pass ended on (frame 0, cell-sorted at the start of its step)
f = sim.cur_substep_local
out = torch.zeros(1, dtype=torch.float32, device=sim.device)
tgt, phi = mom.tgt4[0], mom.sdf[0]
mask = sim.material_row_mask(M.WATER)
sim.reset_grad()
for _ in range(3):
    sim.momentum_loss(mom._mass, tgt, phi, mom.w_density, mom.w_sdf, mom.w_momentum, mask, out, f)
    sim.add_grad_momentum(mom._mass, tgt, phi, mom.w_density, mom.w_sdf, mom.w_momentum, mask, f)
torch.cuda.synchronize()
ev = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
ev[0].record()
for _ in range(args.launches):
    sim.momentum_loss(mom._mass, tgt, phi, mom.w_density, mom.w_sdf, mom.w_momentum, mask, out, f)
ev[1].record()
for _ in range(args.launches):
    sim.add_grad_momentum(mom._mass, tgt, phi, mom.w_density, mom.w_sdf, mom.w_momentum, mask, f)
ev[2].record(); torch.cuda.synchronize()
call_us = dict(fmpm_loss_momentum=ev[0].elapsed_time(ev[1]) * 1e3 / args.launches, fmpm_loss_momentum_grad=ev[1].elapsed_time(ev[2]) * 1e3 / args.launches)
from torch.profiler import profile, ProfilerActivity  # noqa: E402
TAGS = ('k_loss_momentum_deposit', 'k_loss_momentum_node<false>', 'k_loss_momentum_node<true>', 'k_loss_momentum_grad<false>', 'k_loss_momentum_grad<true>',
        'k_loss_density_deposit', 'k_fwd')


def kernel_times(frame, fwd_step):
    """mean device time per launch (us) of the momentum kernels over --launches calls of both entry points on `frame`, of the density deposit
    over as many density_loss calls (and of k_fwd over one forward step from the initial state when fwd_step)"""
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(args.launches):
            sim.momentum_loss(mom._mass, tgt, phi, mom.w_density, mom.w_sdf, mom.w_momentum, mask, out, frame)
            sim.add_grad_momentum(mom._mass, tgt, phi, mom.w_density, mom.w_sdf, mom.w_momentum, mask, frame)
            sim.density_loss(dens._mass, dens.tgt[0], phi, dens.w_density, dens.w_sdf, mask, out, frame)
        if fwd_step:
            env.step()
        torch.cuda.synchronize()
    kern = {}
    for e in prof.key_averages():
        for tag in TAGS:
            if tag in e.key and e.count > 0:
                d = kern.setdefault(tag, [0.0, 0])
                d[0] += getattr(e, 'device_time_total', None) or getattr(e, 'cuda_time_total', 0.0); d[1] += e.count
    return {k: v[0] / v[1] for k, v in kern.items()}


kernel_us = kernel_times(f, False)   # the frame of the timed calls above: cell-sorted at the start of its chunk, as in the training pass
env.loss = None
env.set_state(init, grad_enabled=False)   # frame 0 in the particles' original order: no cell sort
kernel_us_unsorted = kernel_times(0, True)
gpu = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader', '-i', str(sim.device.index or 0)],
                     capture_output=True, text=True).stdout.strip()
med = {k: float(np.median(v)) for k, v in runs.items()}
print(json.dumps(dict(gpu=gpu, steps=steps, particles=N, n_grid=n, median_ms=med, range_ms={k: [min(v), max(v)] for k, v in runs.items()}, runs_ms=runs,
                      ratio_density_over_shape=med['density'] / med['shape'], ratio_momentum_over_shape=med['momentum'] / med['shape'],
                      ratio_momentum_over_density=med['momentum'] / med['density'], per_call_us=call_us, per_kernel_us_sorted=kernel_us, per_kernel_us_unsorted=kernel_us_unsorted,
                      momentum_loss_total=total, finite=bool(np.isfinite(total)))))
