"""allrank_b200 -- H100-native (sm_90a) scoring + listwise-loss + metric path behind allRank's call surfaces.

    from allrank_b200 import losses, metrics          # same names/signatures as allrank.models.{losses,metrics}
    from allrank_b200.model import make_model         # same surface as allrank.models.model.make_model

Importing the package does not load the CUDA library; the first kernel call does, and raises if
liballrank_b200.so has not been built (python -m allrank_b200.build).
"""
__version__ = "0.1.0"
