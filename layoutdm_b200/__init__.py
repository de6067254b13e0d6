"""layoutdm_b200 -- H100-native (sm_90a) implementation of LayoutDM's discrete-diffusion sampling loop.

Host-side mirror of the reference's class API (LayoutDM.sample / BaseMaskAndReplaceDiffusion.sample /
_sample_single_step) on top of the C ABI in include/ldm_b200.h.  See DESIGN.md and INTEGRATION.md."""
from .vocab import Vocab, timestep_plan, decode_ids, refinement_table, linear_centers  # noqa: F401
from .engine import Engine  # noqa: F401
from .diffusion import FusedMaskAndReplaceDiffusion, LayoutDMB200, patch_reference_model  # noqa: F401

__all__ = ["Vocab", "Engine", "FusedMaskAndReplaceDiffusion", "LayoutDMB200", "patch_reference_model", "timestep_plan",
           "decode_ids", "refinement_table", "linear_centers"]
