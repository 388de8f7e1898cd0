"""Pins the restatement of diffusers' EulerDiscreteScheduler (oracle/euler.py) to REAL diffusers under the
stable-diffusion-xl-base-1.0 scheduler config — whenever `import diffusers` works on the machine running the tests.
Elsewhere these tests SKIP, loudly, and the Euler schedule's parity with diffusers stays unpinned, as DDIM's does
(tests/test_oracle_diffusers_pin.py).  CPU only.
"""
import pytest
import torch

diffusers = pytest.importorskip(
    "diffusers", reason="PARITY UNPINNED for the Euler scheduler: `diffusers` is not installed on this machine (it is "
                        "an unvendored, unpinned dependency of the reference); install it to turn oracle/euler.py "
                        "from a restatement into a checked one")

from oracle.euler import EulerSchedule  # noqa: E402
from test_euler_host import SDXL_EULER  # noqa: E402


def _ref():
    from diffusers import EulerDiscreteScheduler
    return EulerDiscreteScheduler.from_config({k: v for k, v in SDXL_EULER.items() if not k.startswith("_")})


@pytest.mark.parametrize("n", [20, 30, 50])
def test_oracle_euler_schedule_matches_diffusers(n):
    ref, mine = _ref(), EulerSchedule()
    ref.set_timesteps(n)
    assert [int(t) for t in ref.timesteps] == mine.set_timesteps(n)
    assert torch.equal(ref.sigmas.float(), mine.sigmas)
    assert float(ref.init_noise_sigma) == mine.init_noise_sigma


@pytest.mark.parametrize("n", [20, 30, 50])
def test_oracle_euler_step_matches_diffusers(n):
    ref, mine = _ref(), EulerSchedule()
    ref.set_timesteps(n)
    mine.set_timesteps(n)
    g = torch.Generator().manual_seed(n)
    x = torch.randn(1, 4, 8, 8, generator=g) * mine.init_noise_sigma
    for i, t in enumerate(ref.timesteps):              # diffusers tracks the step index: walk every step in order
        eps = torch.randn(1, 4, 8, 8, generator=g)
        assert torch.allclose(ref.scale_model_input(x, t), mine.scale_model_input(x, int(t)), rtol=1e-6, atol=0)
        want = ref.step(eps, t, x, return_dict=False)[0]
        got = mine.step(eps, int(t), x)
        assert torch.allclose(got, want, rtol=1e-5, atol=1e-5), i
        x = want
