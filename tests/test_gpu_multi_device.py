"""Several devices in one process: the library's per-device host state (each device's SM count and the tensor-core
kernels' shared-memory opt-ins) must be set up on every device a process uses, not only on the first.  A fresh child
process runs a bf16 MipNerf.forward and a fused bf16 training step on cuda:0, then the same seeded calls on cuda:1;
both devices must succeed and give equal outputs."""
import os
import subprocess
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))


def _outputs(dev):
    import mipnerf_pl_b200 as mp
    from mipnerf_pl_b200.weights import make_state_dict

    b = 300
    rays = mp.namedtuple_map(lambda t: t.to(dev), mp.random_ray_batch(b, seed=5, multiscale=True))
    rgbs = torch.rand(b, 3, generator=torch.Generator().manual_seed(6)).to(dev)
    model = mp.MipNerf(precision="bf16")
    model.load_state_dict(make_state_dict(seed=3, kind="trained_like"))
    model = model.to(dev)
    with torch.no_grad():
        fwd = [t for level in model(rays, False, True) for t in level]
    step = mp.forward_backward(model, rays, rgbs, False, True)
    grads = [p.grad for p in model.parameters()]
    torch.cuda.synchronize(dev)
    return [t.cpu() for t in fwd + [step["loss"]] + grads]


def _child(out):
    sys.path.insert(0, ROOT)
    torch.save([_outputs(torch.device("cuda", i)) for i in (0, 1)], out)


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_bf16_forward_and_training_step_on_two_devices_in_one_process(tmp_path):
    out = str(tmp_path / "outputs.pt")
    r = subprocess.run([sys.executable, __file__, out], cwd=ROOT, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-4000:] + r.stderr[-4000:]
    on0, on1 = torch.load(out)
    assert len(on0) == len(on1)
    for i, (a, b) in enumerate(zip(on0, on1)):
        assert torch.equal(a, b), f"output {i} differs between cuda:0 and cuda:1"


if __name__ == "__main__":
    _child(sys.argv[1])
