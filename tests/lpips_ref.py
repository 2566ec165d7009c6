"""The reference's own LPIPS module (lpipsPyTorch, copied into oracle/_ref/s3g_ref by oracle/build_ref_lpips.sh), built
with seeded weights instead of downloaded ones: torchvision's alexnet is made with weights=None and the lin state dict
comes from the caller.  Test and benchmark infrastructure only."""
from __future__ import annotations

import os
import sys
from unittest import mock

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = os.path.join(ROOT, "oracle", "_ref", "s3g_ref")


def available() -> bool:
    try:
        import torchvision  # noqa: F401
    except ImportError:
        return False
    return os.path.isdir(os.path.join(REF, "lpipsPyTorch"))


def reference_module(features_sd: dict, lin_sd: dict):
    """lpipsPyTorch.modules.lpips.LPIPS('alex', '0.1') with these weights (CPU, float32, eval mode)."""
    import torchvision
    if REF not in sys.path:
        sys.path.insert(0, REF)
    from lpipsPyTorch.modules import lpips as lp_mod, networks
    # utils.get_state_dict's renaming: lin0.model.1.weight -> 0.1.weight
    renamed = {k.replace("lin", "").replace("model.", ""): v for k, v in lin_sd.items()}
    alexnet = torchvision.models.alexnet
    with mock.patch.object(networks.models, "alexnet", lambda *a, **k: alexnet(weights=None)), \
            mock.patch.object(lp_mod, "get_state_dict", lambda *a, **k: renamed):
        m = lp_mod.LPIPS("alex", "0.1")
    m.net.layers.load_state_dict({k[len("features."):]: v for k, v in features_sd.items() if k.startswith("features.")})
    return m.eval()
