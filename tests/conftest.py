import pathlib
import sys

import pytest

ROOT = pathlib.Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
import vlo_bootstrap  # noqa: E402,F401  registers `videollm_online_b200`


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs an H100 (run with -m gpu on a machine that has one)")


@pytest.fixture(scope="session")
def golden():
    import torch
    return torch.load(ROOT / "tests" / "golden" / "tiny_reference.pt", weights_only=False)


@pytest.fixture(scope="session")
def tiny():
    """tiny config + the seeded weights the golden fixtures were generated with"""
    import torch
    from videollm_online_b200 import tiny_config
    from videollm_online_b200 import weights as W
    cfg = tiny_config()
    llm = W.synthetic_llm_state(cfg, seed=0)
    llm["lm_head.weight"] = (llm["lm_head.weight"].float() * 8).to(torch.bfloat16)
    vis = W.synthetic_vision_state(cfg, seed=1)
    return cfg, llm, vis
