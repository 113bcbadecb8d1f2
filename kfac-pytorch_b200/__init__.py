"""H100-native K-FAC hot path: drop-in for kfac.preconditioner.KFACPreconditioner.

Import as `kfac_b200` (the root-level shim package extends its __path__ here;
the directory name `kfac-pytorch_b200` is not a valid Python identifier).
"""
