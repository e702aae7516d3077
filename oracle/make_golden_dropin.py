"""TEST INFRASTRUCTURE — generator of tests/golden/dropin_pose_resnet.json.  Needs the original project's tree
(EPI_REFERENCE_ROOT): builds the UNMODIFIED reference PoseResNet (modeling/backbones/resnet.py:257-305) at the
configs/epipolar/keypoint_h36m_zresidual_fixed.yaml shape and records what a drop-in `Epipolar` must match — the state-dict
names and shapes under `epipolar_sampler.` and the parameter names of the reference `Epipolar.forward`.

    python -m oracle.make_golden_dropin
"""
import importlib
import inspect
import json
import os
import sys
import tempfile
import types
import warnings

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from oracle import ref_harness as rh  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "dropin_pose_resnet.json")
PREFIX = "epipolar_sampler."


def import_reference_resnet():
    warnings.filterwarnings("ignore")
    _, ref_cfg = rh.load_reference()
    import PIL
    if not hasattr(PIL, "PILLOW_VERSION"):               # the reference targets Pillow < 7 (data/transforms/image.py:6)
        PIL.PILLOW_VERSION = PIL.__version__
    R = rh.REFERENCE_ROOT
    for name, sub in (("modeling.backbones", ("modeling", "backbones")), ("data", ("data",)),
                      ("data.transforms", ("data", "transforms")), ("utils", ("utils",))):
        if name not in sys.modules:                      # leaf packages only: modeling/__init__.py pulls the whole model zoo
            pkg = types.ModuleType(name)
            pkg.__path__ = [os.path.join(R, *sub)]
            sys.modules[name] = pkg
    ref_cfg.FOLDER_NAME = tempfile.mkdtemp()             # resnet.py:16 opens a log file there at import time
    return importlib.import_module("modeling.backbones.resnet"), ref_cfg


def main():
    import epipolar_transformers_b200 as epi
    rn, ref_cfg = import_reference_resnet()
    rh.apply_cfg(ref_cfg, epi.cfg_h36m_r50_256())
    ref_cfg.BACKBONE.BODY = "epipolarposeR-50"
    m_ref = rn.PoseResNet(rn.Bottleneck, [3, 4, 6, 3], ref_cfg)
    sd = m_ref.state_dict()
    out = {
        "meta": "reference PoseResNet (epipolarposeR-50, keypoint_h36m_zresidual_fixed shape): its Epipolar sub-module",
        "state_dict": {k[len(PREFIX):]: list(v.shape) for k, v in sd.items() if k.startswith(PREFIX)},
        "forward_params": [p for p in inspect.signature(rn.Epipolar.forward).parameters if p != "self"],
    }
    with open(OUT, "w") as f:
        json.dump(out, f, indent=1, sort_keys=True)
    print("wrote", OUT, len(out["state_dict"]), "tensors")


if __name__ == "__main__":
    main()
