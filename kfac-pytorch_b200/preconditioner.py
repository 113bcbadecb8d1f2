"""Public drop-in class: `KFACPreconditioner(model, **kw).step()`.

Constructor signature, validation order, error messages and derived attributes
follow kfac/preconditioner.py:54-334 so a user of the reference can switch the
import and keep their training script:

    from kfac_b200.preconditioner import KFACPreconditioner
    preconditioner = KFACPreconditioner(model, ...)
    loss.backward(); preconditioner.step(); optimizer.step()
"""
from __future__ import annotations

import logging
import warnings
from typing import Any, Callable

import torch
import torch.distributed as dist

from kfac_b200.assignment import KAISAAssignment
from kfac_b200.base_preconditioner import BaseKFACPreconditioner
from kfac_b200.distributed import ArenaCommunicator, get_rank, get_world_size
from kfac_b200.enums import (AllreduceMethod, AssignmentStrategy, ComputeMethod,
                             DistributedStrategy)
from kfac_b200.layers import register_modules

logger = logging.getLogger(__name__)


def _mock_new_group(x: list[int]) -> None:
    return None


class KFACPreconditioner(BaseKFACPreconditioner):
    """K-FAC gradient preconditioner with KAISA placement on H100 (sm_90a)."""

    def __init__(
        self,
        model: torch.nn.Module,
        *,
        factor_update_steps: Callable[[int], int] | int = 1,
        inv_update_steps: Callable[[int], int] | int = 1,
        damping: Callable[[int], float] | float = 0.001,
        factor_decay: Callable[[int], float] | float = 0.95,
        kl_clip: Callable[[int], float] | float = 0.001,
        lr: Callable[[int], float] | float = 0.1,
        accumulation_steps: int = 1,
        allreduce_bucket_cap_mb: float = 25.0,
        assignment_strategy: AssignmentStrategy | str = AssignmentStrategy.COMPUTE,
        colocate_factors: bool = True,
        compute_method: ComputeMethod | str = ComputeMethod.EIGEN,
        compute_eigenvalue_outer_product: bool = True,
        grad_worker_fraction: DistributedStrategy | float = DistributedStrategy.COMM_OPT,
        symmetry_aware: bool = False,
        grad_scaler: Any | Callable[[], float] | None = None,
        factor_dtype: torch.dtype | None = None,
        inv_dtype: torch.dtype = torch.float32,
        skip_layers: list[str] | None = None,
        update_factors_in_hook: bool = True,
        loglevel: int = logging.DEBUG,
    ) -> None:
        if allreduce_bucket_cap_mb < 0:
            raise ValueError('allreduce_bucket_cap_mb must be >= 0')
        if isinstance(assignment_strategy, str):
            assignment_strategy = AssignmentStrategy[assignment_strategy.upper()]
        if isinstance(compute_method, str):
            compute_method = ComputeMethod[compute_method.upper()]
        if (compute_method == ComputeMethod.EIGEN and compute_eigenvalue_outer_product
                and not colocate_factors):
            raise ValueError('colocate_factors must be True to use compute_eigenvalue_outer_product')
        # factors and second-order data are STORED in float32 arenas (tensor-core 3xTF32 with fp32
        # accumulation has no fp64 path): float64 is accepted and cast at the boundary, half-precision
        # factor dtypes round the hook inputs like the reference does (kfac/layers/base.py:350,364)
        if factor_dtype not in (None, torch.float32, torch.float64, torch.float16, torch.bfloat16):
            raise ValueError(f'unsupported factor_dtype {factor_dtype}')
        if inv_dtype not in (torch.float32, torch.float64):
            raise ValueError(
                'kfac_b200 computes the eigendecompositions and the precondition in float32 (like '
                'kfac/layers/eigen.py:310-312); inv_dtype must be float32 or float64 (cast at the boundary), '
                f'got {inv_dtype}')

        size = get_world_size()
        if isinstance(grad_worker_fraction, DistributedStrategy):
            distributed_strategy = grad_worker_fraction
            if distributed_strategy == DistributedStrategy.COMM_OPT:
                grad_worker_fraction = 1.0
            elif distributed_strategy == DistributedStrategy.HYBRID_OPT:
                grad_worker_fraction = 0.5
            elif distributed_strategy == DistributedStrategy.MEM_OPT:
                grad_worker_fraction = 1.0 / size
            else:
                raise AssertionError(f'Unknown enum {grad_worker_fraction}')
        else:
            if not 0 <= grad_worker_fraction or not 1 >= grad_worker_fraction:
                raise ValueError('grad_worker_fraction must in [0, 1]')
            if grad_worker_fraction == 0:
                grad_worker_fraction = 1.0 / size
            if size % max(1, round(size * grad_worker_fraction)) != 0:
                raise ValueError('grad_worker_fraction must produce groups of equal size')
            if grad_worker_fraction == 1:
                grad_worker_fraction = 1.0
                distributed_strategy = DistributedStrategy.COMM_OPT
            elif grad_worker_fraction <= 1 / size:
                distributed_strategy = DistributedStrategy.MEM_OPT
            else:
                distributed_strategy = DistributedStrategy.HYBRID_OPT
        assert isinstance(grad_worker_fraction, float)

        if not colocate_factors and distributed_strategy is DistributedStrategy.MEM_OPT:
            warnings.warn('grad_worker_frac=1/world_size (MEM_OPT) requires '
                          'colocate_factors=True. Enabling colocate_factors.', stacklevel=2)
            colocate_factors = True

        self.allreduce_bucket_cap_mb = allreduce_bucket_cap_mb
        self.assignment_strategy = assignment_strategy
        self.colocate_factors = colocate_factors
        self.compute_eigenvalue_outer_product = compute_eigenvalue_outer_product
        self.compute_method = compute_method
        self.distributed_strategy = distributed_strategy
        self.grad_worker_fraction = grad_worker_fraction
        self.grad_scaler = grad_scaler
        self.factor_dtype = factor_dtype
        self.inv_dtype = inv_dtype
        self.skip_layers = [] if skip_layers is None else skip_layers
        self.symmetry_aware = symmetry_aware
        self.allreduce_method = (AllreduceMethod.ALLREDUCE_BUCKETED if allreduce_bucket_cap_mb > 0
                                 else AllreduceMethod.ALLREDUCE)
        self.tdc = ArenaCommunicator(bucket_cap_mb=allreduce_bucket_cap_mb)

        kfac_layers = register_modules(
            model, self.skip_layers, method=compute_method,
            prediv_eigenvalues=compute_eigenvalue_outer_product, grad_scaler=grad_scaler,
            factor_dtype=factor_dtype, inv_dtype=inv_dtype, symmetry_aware=symmetry_aware)
        for name, kfac_layer in kfac_layers.values():
            logger.log(loglevel, f'Registered name="{name}": {repr(kfac_layer)}')

        if assignment_strategy == AssignmentStrategy.COMPUTE:
            cost = lambda n: n ** 3  # noqa: E731
        elif assignment_strategy == AssignmentStrategy.MEMORY:
            cost = lambda n: n ** 2  # noqa: E731
        else:
            raise AssertionError(f'Unknown assignment_strategy={assignment_strategy}')
        work = {name: {'A': cost(l.a_dim), 'G': cost(l.g_dim)} for name, l in kfac_layers.values()}

        assignment = KAISAAssignment(
            work, local_rank=get_rank(), world_size=size,
            grad_worker_fraction=grad_worker_fraction,
            group_func=dist.new_group if dist.is_initialized() else _mock_new_group,
            colocate_factors=colocate_factors)
        logger.log(loglevel, f'KFAC layer assignments: {assignment}')

        defaults = {
            'allreduce_bucket_cap_mb': allreduce_bucket_cap_mb,
            'allreduce_method': self.allreduce_method,
            'assignment_strategy': assignment_strategy,
            'colocate_factors': colocate_factors,
            'compute_eigenvalue_outer_product': compute_eigenvalue_outer_product,
            'compute_method': compute_method,
            'distributed_strategy': distributed_strategy,
            'grad_worker_fraction': grad_worker_fraction,
            'grad_scaler': grad_scaler is not None,
            'factor_dtype': factor_dtype,
            'inv_dtype': inv_dtype,
            'skip_layers': self.skip_layers,
            'symmetry_aware': symmetry_aware,
        }
        super().__init__(
            kfac_layers, factor_update_steps=factor_update_steps,
            inv_update_steps=inv_update_steps, factor_decay=factor_decay, damping=damping,
            kl_clip=kl_clip, lr=lr, accumulation_steps=accumulation_steps,
            assignment=assignment, update_factors_in_hook=update_factors_in_hook,
            defaults=defaults, tdc=self.tdc, loglevel=loglevel)
