"""CPU: the drop-in really drops in.  The reference PoseResNet (modeling/backbones/resnet.py:257-305 of the original project)
builds its `epipolar_sampler` from the name `Epipolar`; INTEGRATION.md section 2 re-binds that name to ours.  What the
re-bound module must match was recorded from the unmodified reference model (oracle/make_golden_dropin.py) in
tests/golden/dropin_pose_resnet.json: the state-dict names and shapes under `epipolar_sampler.` and the parameter names of
`Epipolar.forward`.  A reference state dict of those shapes must load strictly into ours."""
import inspect
import json
import os

import torch

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "dropin_pose_resnet.json")


def test_epipolar_drops_into_reference_pose_resnet():
    import epipolar_transformers_b200 as epi
    ref = json.load(open(GOLDEN))
    m = epi.Epipolar(cfg=epi.cfg_h36m_r50_256())          # configs/epipolar/keypoint_h36m_zresidual_fixed.yaml shape
    ours = m.state_dict()
    assert set(ours) == set(ref["state_dict"])                           # identical parameter / buffer names
    for k, shape in ref["state_dict"].items():
        assert tuple(ours[k].shape) == tuple(shape), k
    g = torch.Generator().manual_seed(0)
    sd = {k: (torch.tensor(7) if k.endswith("num_batches_tracked") else torch.randn(shape, generator=g))
          for k, shape in ref["state_dict"].items()}
    res = m.load_state_dict(sd, strict=True)
    assert not res.missing_keys and not res.unexpected_keys
    assert torch.equal(m.state_dict()["z.weight"], sd["z.weight"])
    # the forward signature the caller uses (resnet.py:385-387): positional feats/KRTs + camera kwargs
    params = [p for p in inspect.signature(m.forward).parameters if p != "self"]
    assert params == ref["forward_params"]
