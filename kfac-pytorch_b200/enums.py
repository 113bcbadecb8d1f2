"""Constructor enums of the drop-in API (mirror of kfac/enums.py:8-54: same
names and member values so `kfac.enums.X.Y.name` strings round-trip)."""
from __future__ import annotations

from enum import Enum


class AllreduceMethod(Enum):
    ALLREDUCE = 1
    ALLREDUCE_BUCKETED = 2


class AssignmentStrategy(Enum):
    """Cost heuristic of the greedy layer placement: n^3 (COMPUTE) / n^2 (MEMORY)."""
    COMPUTE = 1
    MEMORY = 2


class ComputeMethod(Enum):
    """EIGEN: (G (x) A + damping I)^-1 ;  INVERSE: (G+damping I)^-1 (x) (A+damping I)^-1 ;
    EKFAC: the eigenbases of EIGEN with second moments S measured in them in place of dg (x) da
    (George et al., 2018; an extension beyond the reference)."""
    EIGEN = 1
    INVERSE = 2
    EKFAC = 3


class DistributedStrategy(Enum):
    """KAISA shortcuts: grad_worker_fraction = 1, 1/world_size, 1/2."""
    COMM_OPT = 1
    MEM_OPT = 2
    HYBRID_OPT = 3
