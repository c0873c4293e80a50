"""cornac_b200 -- H100 (sm_90a) implementation of Cornac's BPR / MF train-and-rank hot path.

    from cornac_b200 import BPR, MF, PMF, NMF   # drop-in for cornac.models.BPR / MF / PMF / NMF
    from cornac_b200 import SoRec, MCF          # ... and the graph co-factorisations cornac.models.SoRec / MCF
    cornac.Experiment(eval_method=..., models=[BPR(k=64, ...)], metrics=[...]).run()

Layers:  include/b200cornac.h (C ABI)  <-  cornac_b200/csrc (CUDA)  <-  cornac_b200.engine
(ctypes, device tensors)  <-  cornac_b200.recom_bpr / recom_mf (cornac.models.Recommender
plug-ins).  The plug-in classes need the `cornac` package importable (they subclass its
Recommender so that cornac.Experiment accepts them); the engine does not.
"""
__all__ = ["BPR", "WBPR", "MMMF", "VEBPR", "SBPR", "MF", "WMF", "BaselineOnly", "UserKNN", "ItemKNN", "PMF", "NMF", "EASE", "HPF", "SoRec", "MCF", "C2PF", "EFM", "MTER", "engine", "B200Error"]

from ._lib import B200Error  # noqa: F401


def __getattr__(name):
    if name == "BPR":
        from .recom_bpr import BPR
        return BPR
    if name == "WBPR":
        from .recom_bpr import WBPR
        return WBPR
    if name == "MMMF":
        from .recom_bpr import MMMF
        return MMMF
    if name == "VEBPR":
        from .recom_bprx import VEBPR
        return VEBPR
    if name == "SBPR":
        from .recom_bprx import SBPR
        return SBPR
    if name == "MF":
        from .recom_mf import MF
        return MF
    if name == "WMF":
        from .recom_wmf import WMF
        return WMF
    if name in ("UserKNN", "ItemKNN"):
        from . import recom_knn
        return getattr(recom_knn, name)
    if name == "PMF":
        from .recom_pmf import PMF
        return PMF
    if name == "NMF":
        from .recom_nmf import NMF
        return NMF
    if name == "EASE":
        from .recom_ease import EASE
        return EASE
    if name == "HPF":
        from .recom_hpf import HPF
        return HPF
    if name == "SoRec":
        from .recom_sorec import SoRec
        return SoRec
    if name == "MCF":
        from .recom_mcf import MCF
        return MCF
    if name == "C2PF":
        from .recom_c2pf import C2PF
        return C2PF
    if name == "EFM":
        from .recom_efm import EFM
        return EFM
    if name == "MTER":
        from .recom_mter import MTER
        return MTER
    if name == "BaselineOnly":
        from .recom_bo import BaselineOnly
        return BaselineOnly
    if name == "engine":
        import importlib
        return importlib.import_module(".engine", __name__)
    raise AttributeError(name)
