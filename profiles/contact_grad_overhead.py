"""Cost of the contact-parameter gradients (MPMSimulator.param_grad: static / rigid friction, rigid softness, restitution) on a contact-heavy
scene: 262,144 ICECREAM particles at 64^3 on the floor of a cube with restitution 0.3, a static box collider on the grid and a soft Rigid box
(friction 8, softness 100) colliding at particle level, pushed by a small action every step.  One forward + backward pass of --steps steps,
timed with CUDA events, in three modes alternated run by run so that all see the same machine state: param_grad off, material gradients only
(the contact accumulator unbound), material + contact.  Prints one JSON line with the medians, the ranges, and the card and its power limit.
    python profiles/contact_grad_overhead.py [--steps 10] [--runs 5]"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))
from conftest import make_particles, box_sdf  # noqa: E402
from fluidlab_b200 import TaichiEnv, macros as M, _lib  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument('--steps', type=int, default=10)
ap.add_argument('--runs', type=int, default=5)
args = ap.parse_args()
assert torch.cuda.is_available(), 'needs a CUDA device'
n_grid, N, steps = 64, 262144, args.steps
rng = np.random.RandomState(17)
P = make_particles(rng.uniform((0.3, 0.205, 0.3), (0.7, 0.45, 0.7), size=(N, 3)), M.ICECREAM, n_grid)
env = TaichiEnv(quality=n_grid / 64, max_substeps_local=10 * steps + 10, gravity=(0.0, -10.0, 0.0), horizon=steps + 1)
sim = env.simulator
vox, T = box_sdf((0.06, 0.06, 0.15), 0.2)
env.setup_agent(dict(type='AgentRigid', params=dict(collide_type='particle'), effectors=[dict(
    type='Rigid', params=dict(init_pos=(0.28, 0.4, 0.5), init_euler=(0.0, 0.0, 0.0), action_dim=3),
    mesh=dict(file='box.obj', material=M.STIRRER, softness=100.0, sdf=dict(voxels=vox, T_mesh_to_voxels=T)),
    boundary=dict(type='cube', lower=(0.05,) * 3, upper=(0.95,) * 3))]))
env.setup_boundary(type='cube', lower=(0.2, 0.2, 0.2), upper=(0.8, 0.8, 0.8), restitution=0.3)
bv, bT = box_sdf((0.12, 0.02, 0.12), 0.3)
env.add_static(file='box.obj', material=M.CUP, has_dynamics=True, pos=(0.6, 0.24, 0.5), sdf=dict(voxels=bv, T_mesh_to_voxels=bT))
env.particle_bodies.get = lambda: P
env.build()
sim.set_contact_params(rigid_friction=8.0)
st0 = sim.get_state()
action = np.array([0.004, -0.002, 0.0], dtype=np.float32)
zero3, zero9 = np.zeros((N, 3), np.float32), np.zeros((N, 3, 3), np.float32)
seed = np.tile(np.array([1.0, 1.0, 0.5], dtype=np.float32), (N, 1))


def fwd_bwd(mode):
    sim.param_grad = mode != 'off'
    env.set_state(st0, grad_enabled=True)
    env.apply_agent_action_p(np.array([0.28, 0.4, 0.5], dtype=np.float32))
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(steps):
        env.step(action)
    env.reset_grad()   # binds / unbinds both accumulators with param_grad
    if mode == 'material':
        assert sim._lib.fmpm_set_contact_grad(sim._h, None) == 0
    elif mode == 'contact':
        cg = _lib.FmpmContactGrad(); cg.gcontact = sim._gcontact.data_ptr()
        assert sim._lib.fmpm_set_contact_grad(sim._h, C.byref(cg)) == 0
    sim.set_grad(seed, zero3, zero9, zero9)
    for _ in range(steps):
        env.step_grad(action)
    b.record(); torch.cuda.synchronize()
    return a.elapsed_time(b)


modes = ('off', 'material', 'contact')
for m in modes:
    fwd_bwd(m)   # warm-up
runs = {m: [] for m in modes}
for _ in range(args.runs):
    for m in modes:
        runs[m].append(fwd_bwd(m))
g = sim.get_param_grad()
gpu = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader', '-i', str(sim.device.index or 0)],
                     capture_output=True, text=True).stdout.strip()
med = {m: float(np.median(runs[m])) for m in modes}
print(json.dumps(dict(gpu=gpu, steps=steps, particles=N, median_ms=med, range_ms={m: [min(runs[m]), max(runs[m])] for m in modes}, runs_ms=runs,
                      ratio_material_over_off=med['material'] / med['off'], ratio_contact_over_material=med['contact'] / med['material'],
                      contact_grad={k: (v.tolist() if hasattr(v, 'tolist') else v) for k, v in g.items() if k not in ('mu', 'lam', 'rho', 'gravity')})))
