"""CPU tier: the phased ROMix instances compiled into label_kernels.cu's launch table are exactly the ones
test_gpu_romix_phased.py runs against the oracle."""
import importlib.util
import re
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
SRC = (ROOT / "go-spacemesh_b200" / "csrc" / "label_kernels.cu").read_text()


def _body(signature):
    i = SRC.index(signature)
    return SRC[i: SRC.index("\n}\n", i)]


def test_phased_instances_are_all_in_the_matrix():
    spec = importlib.util.spec_from_file_location("romix_phased", Path(__file__).with_name("test_gpu_romix_phased.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    cases = re.findall(r"case (\d+): return romix_phased_kernel<MW, (\d+)>;", _body("static romix_fn pick_phased_tpb("))
    assert cases and all(t == t2 for t, t2 in cases)
    masks = {int(x) for x in re.findall(r"X\((\d+)\)", re.search(r"#define B200POST_MW_LIST\(X\)(.*)", SRC).group(1))}
    compiled = {(mw, int(t)) for mw in masks for t, _ in cases}
    assert len(mod.PHASED_MATRIX) == len(set(mod.PHASED_MATRIX))
    assert set(mod.PHASED_MATRIX) == compiled
    # the phased kernel is only reached through its own table: the classic table (pick) does not list it
    assert "ROMIX_PHASED" not in _body("static romix_fn pick(")
