"""CPU: a user model compiled with NVRTC carries the single-GPU LL form of its split-cost kernel.

mppi_user_model_register looks that kernel up under one unmangled name whenever the module has a split-cost kernel, so
every module with one must export it; a model with copies > 1 has neither."""
import torch

from tests import ensemble_models, user_models

LL_NAME = b"mppi_user_fused_command_kernel_ll"


def test_user_module_exports_the_ll_kernel_beside_its_split_cost_kernel():
    cubin, names = user_models.pendulum_user_model().compile_rtc(torch.float32, 0)
    assert names[1] is not None and LL_NAME in cubin


def test_module_without_split_cost_kernel_has_no_ll_kernel():
    model, dtype, variant = ensemble_models.prebuilt()[0]
    assert model.copies > 1
    cubin, names = model.compile_rtc(dtype, variant)
    assert names[1] is None and LL_NAME not in cubin
