"""gcbfplus.algo surface (gcbfplus/algo/__init__.py:1-18)."""
from .base import MultiAgentController
from .cbf_qp import CentralizedCBF, DecShareCBF
from .gcbf_plus import GCBFPlus


def make_algo(algo: str, **kwargs) -> MultiAgentController:
    """gcbfplus/algo/__init__.py:8-18.  GCBF-v0 ('gcbf') is outside the scope of this project (SURVEY 2)."""
    if algo == "gcbf+":
        return GCBFPlus(**kwargs)
    if algo == "centralized_cbf":
        return CentralizedCBF(**kwargs)
    if algo == "dec_share_cbf":
        return DecShareCBF(**kwargs)
    if algo == "gcbf":
        raise NotImplementedError(f"algo '{algo}' is outside the CUDA hot-path scope (SURVEY.md section 2, row 12)")
    raise ValueError(f"Unknown algorithm: {algo}")
