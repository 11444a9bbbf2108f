"""``dataset/expl_hdf5.py`` of the reference: the reader of ``results.hdf5`` (see ``perturbation.ImagenetResults``)."""
from transformer_explainability_b200.perturbation import ImagenetResults

__all__ = ["ImagenetResults"]
