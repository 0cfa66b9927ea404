"""fluidlab_b200 — CUDA-native (H100, sm_90a) MLS-MPM substep behind FluidLab's FluidEngine simulator API.

Hot path in libfluidmpm.so (hand-written CUDA, C ABI: include/fluidmpm.h); this package is the thin Python host
mirroring fluidlab.fluidengine: `MPMSimulator`, `TaichiEnv`, agents/effectors, losses, boundaries, bodies."""
from .macros import *  # noqa: F401,F403
from .simulator import MPMSimulator  # noqa: F401
from .taichi_env import TaichiEnv  # noqa: F401
from .bodies import Bodies  # noqa: F401
from .boundaries import create_boundary  # noqa: F401
from .agents import Agent, AgentInjector, AgentRigid, AgentIceCreamDynamic, AgentPouring, AgentJetBot, AgentCirculation  # noqa: F401
from .effectors import Effector, Injector, BallInjector, Rigid, AirCon  # noqa: F401
from .smoke import SmokeField  # noqa: F401
from .meshes import Static, Dynamic, Statics  # noqa: F401
from .losses import Loss, ShapeMatchingLoss, DensityMatchingLoss, MomentumMatchingLoss, LatteArtLoss, CirculationLoss, IceCreamDynamicLoss, IceCreamStaticLoss  # noqa: F401
from .optimizer import (Adam, ActionsPolicy, TrainablePolicy, LatteArtPolicy, LatteArtStirPolicy, IceCreamDynamicPolicy, IceCreamStaticPolicy,  # noqa: F401
                        CirculationPolicy, PouringPolicy, TransportingPolicy, GatheringPolicy, GatheringOPolicy, MixingPolicy, Solver, forward_backward, trainable_policy)
