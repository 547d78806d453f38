"""The committed wgmma width wrappers (csrc/nn_wgmma_n.cuh) are what tools/gen_wgmma.py produces."""
import importlib.util
import os

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_wgmma_header_is_generated():
    spec = importlib.util.spec_from_file_location("gen_wgmma", os.path.join(ROOT, "tools", "gen_wgmma.py"))
    gen = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(gen)
    with open(gen.OUT) as f:
        assert f.read() == gen.render(), "re-run python tools/gen_wgmma.py"
