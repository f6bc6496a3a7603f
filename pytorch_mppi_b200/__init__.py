"""pytorch_mppi_b200 — H100-native MPPI rollout-and-reweight engine with the API of
UM-ARM-Lab/pytorch_mppi (`MPPI`, `SMPPI`, `KMPPI`, `command()`, dynamics/running_cost plugins)."""
from .mppi import (MPPI, SMPPI, KMPPI, MPPI_Batched, RBFKernel, TimeKernel, SpecificActionSampler, run_mppi,  # noqa: F401
                   ClosedLoopResult)
from .models import Pendulum, LinearPoint, PendulumMLP, PendulumMLPEnsemble, CudaModel, AnalyticModel  # noqa: F401

__all__ = ["MPPI", "SMPPI", "KMPPI", "MPPI_Batched", "RBFKernel", "TimeKernel", "SpecificActionSampler", "run_mppi",
           "ClosedLoopResult", "Pendulum", "LinearPoint", "PendulumMLP", "PendulumMLPEnsemble", "CudaModel", "AnalyticModel"]
