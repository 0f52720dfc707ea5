"""CPU tier: the ROMix instances compiled into the launch table of label_kernels.cu are exactly the ones the GPU matrix
(test_gpu_romix_matrix.py) runs, so that an instance added to the table without a test fails here."""
import importlib.util
import re
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
SRC = (ROOT / "go-spacemesh_b200" / "csrc" / "label_kernels.cu").read_text()


def _matrix():
    spec = importlib.util.spec_from_file_location("romix_matrix", Path(__file__).with_name("test_gpu_romix_matrix.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def _body(signature):
    """the text of the function whose definition starts with `signature`, up to its closing brace at column 0"""
    i = SRC.index(signature)
    return SRC[i: SRC.index("\n}\n", i)]


def _masks():
    m = re.search(r"#define B200POST_MW_LIST\(X\)(.*)", SRC)
    return {int(x) for x in re.findall(r"X\((\d+)\)", m.group(1))}


def test_pipelined_instances_are_all_in_the_matrix():
    body = _body("static pipe_fn pick_pipe_tpb(")
    # `case T: return romix_pipe_kernel<MW, T, DR>;` under each dr_unroll branch, for every MW of the mask list
    cases = re.findall(r"case (\d+): return romix_pipe_kernel<MW, (\d+), (\d+)>;", body)
    assert cases and all(t == t2 for t, t2, _ in cases)
    compiled = {(mw, int(t), int(dr)) for mw in _masks() for t, _, dr in cases}
    matrix = _matrix().PIPE_MATRIX
    assert len(matrix) == len(set(matrix))
    assert set(matrix) == compiled
    assert len(compiled) == 16


def test_classic_instances_are_all_in_the_matrix():
    tpbs = {int(t) for t, t2 in re.findall(r"case (\d+): return romix_kernel<VARIANT, MW, (\d+)>;",
                                           _body("static romix_fn pick_tpb("))}
    variants = re.findall(r"case ROMIX_(\w+): return pick_mw<ROMIX_\1>", _body("static romix_fn pick("))
    assert set(variants) == {"DIRECT", "COALESCED", "BULK", "NOMEM"}
    numbers = {name: int(v) for name, v in re.findall(r"ROMIX_(\w+)\s*=\s*(\d+)",
                                                      (ROOT / "go-spacemesh_b200" / "csrc" / "label_kernels.cuh").read_text())}
    # ROMIX_NOMEM skips the scratchpad: its output is not a label, so it has no place in a parity matrix
    compiled = {(numbers[v], mw, t) for v in variants if v != "NOMEM" for mw in _masks() for t in tpbs}
    matrix = _matrix().CLASSIC_MATRIX
    assert len(matrix) == len(set(matrix))
    assert set(matrix) == compiled


def test_low_latency_instances_are_all_in_the_matrix():
    body = _body("cudaError_t launch_romix_lowlat(")
    compiled = {int(m) for m in re.findall(r"romix_lowlat_kernel<(\d+)><<<", body)}
    assert compiled == _masks() == set(_matrix().LOWLAT_MASKS)
