"""CPU: the choice of the tensor-core operand splits (DESIGN §4.2) pinned by emulation -- exact products of the split operands, fp32
accumulation, the test MLP weights, 20,000 interpolated feature vectors, against float64.  bf16x3 must be fp32-level, the inference
default f16w2 must hold the north-star bar of 1e-4 per sample with margin, and the cheaper bf16 split must NOT (that is why it is
not offered)."""
import importlib.util
from pathlib import Path


def test_operand_split_errors():
    spec = importlib.util.spec_from_file_location("split_accuracy", Path(__file__).resolve().parents[1] / "tools" / "split_accuracy.py")
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    err = {k.split(":")[0].split(" (")[0]: v for k, v in mod.errors().items()}
    assert err["bf16x3"][0] < 2e-6 and err["bf16x3"][1] < 1e-6
    assert err["f16w2"][0] < 5e-5 and err["f16w2"][1] < 2e-5          # 1e-4 bar with a factor > 2 to spare
    assert err["bf16x2"][0] > 1e-4                                      # two bf16 MMAs do not hold the bar
    assert err["fp16x3"][0] < err["bf16x3"][0]                          # (for the record: fp16 halves would be more accurate than bf16 halves)


def test_operand_split_errors_on_the_surface_network():
    """the opaque surface network (synthetic.surface_scene, densities up to 250 at sharpness 1000): f16w2's error is relative to the
    activations -- ~5e-4 of sigma, ~2e-4 on colour, inside the bars of tests/test_gpu_opaque.py -- while bf16x3 stays fp32-level"""
    spec = importlib.util.spec_from_file_location("split_accuracy", Path(__file__).resolve().parents[1] / "tools" / "split_accuracy.py")
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    err = {k.split(":")[0].split(" (")[0]: v for k, v in mod.errors(*mod.surface_inputs(1000)).items()}
    assert err["bf16x3"][4] < 2e-5 and err["bf16x3"][1] < 1e-5
    assert 2e-4 < err["f16w2"][4] < 1e-3 and err["f16w2"][1] < 3e-4
