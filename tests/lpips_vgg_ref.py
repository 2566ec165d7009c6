"""The reference's own LPIPS module with the VGG16 backbone, built as lpips_ref.py builds the AlexNet one: torchvision's
vgg16 is made with weights=None, the lin state dict comes from the caller and the seeded features are loaded into it.
Test and benchmark infrastructure only."""
from __future__ import annotations

import sys
from unittest import mock

from lpips_ref import REF, available  # noqa: F401


def reference_module(features_sd: dict, lin_sd: dict):
    """lpipsPyTorch.modules.lpips.LPIPS('vgg', '0.1') with these weights (CPU, float32, eval mode)."""
    import torchvision
    if REF not in sys.path:
        sys.path.insert(0, REF)
    from lpipsPyTorch.modules import lpips as lp_mod, networks
    # utils.get_state_dict's renaming: lin0.model.1.weight -> 0.1.weight
    renamed = {k.replace("lin", "").replace("model.", ""): v for k, v in lin_sd.items()}
    vgg16 = torchvision.models.vgg16
    with mock.patch.object(networks.models, "vgg16", lambda *a, **k: vgg16(weights=None)), \
            mock.patch.object(lp_mod, "get_state_dict", lambda *a, **k: renamed):
        m = lp_mod.LPIPS("vgg", "0.1")
    # vgg16().features also holds the ReLUs and max-pools (no parameters): the convolutions' keys are all of its state
    m.net.layers.load_state_dict({k[len("features."):]: v for k, v in features_sd.items() if k.startswith("features.")})
    return m.eval()
