"""CPU tier: the phased ROMix instances compiled into label_kernels.cu's launch table are exactly the ones
test_gpu_romix_phased.py and test_gpu_romix_phased_matrix.py run against the oracle."""
import importlib.util
import re
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
SRC = (ROOT / "go-spacemesh_b200" / "csrc" / "label_kernels.cu").read_text()


def _body(signature):
    i = SRC.index(signature)
    return SRC[i: SRC.index("\n}\n", i)]


def _matrix(module):
    spec = importlib.util.spec_from_file_location(module, Path(__file__).with_name(module + ".py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod.PHASED_MATRIX


def test_phased_instances_are_all_in_the_matrix():
    cases = re.findall(r"case (\d+): return romix_phased_kernel<MW, (\d+)>;", _body("static romix_fn pick_phased_tpb("))
    assert cases and all(t == t2 for t, t2 in cases)
    masks = {int(x) for x in re.findall(r"X\((\d+)\)", re.search(r"#define B200POST_MW_LIST\(X\)(.*)", SRC).group(1))}
    compiled = {(mw, int(t)) for mw in masks for t, _ in cases}
    for module in ("test_gpu_romix_phased", "test_gpu_romix_phased_matrix"):
        matrix = _matrix(module)
        assert len(matrix) == len(set(matrix)), module
        assert set(matrix) == compiled, module
    # the phased kernel is only reached through its own table: the classic table (pick) does not list it
    assert "ROMIX_PHASED" not in _body("static romix_fn pick(")
