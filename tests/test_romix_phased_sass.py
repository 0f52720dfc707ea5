"""CPU tier: what ptxas makes of romix_phased_kernel, the default ROMix layer.  Compiles label_kernels.cu for sm_90a and
checks, from -Xptxas -v and cuobjdump -sass:
  - every instance fits in 127 registers with no spills;
  - the step loops (the bodies of the conditional backward branches) hold no SHFL and no WARPSYNC / ENDCOLLECTIVE: the
    row indices of the mix requests pass through shared memory, and the collective sequences ptxas emits for
    __syncwarp stay in the out-of-line divergent fall-backs;
  - a fill loop stores each tile with one TMA bulk store (UBLKCP) and has no STG;
  - few instructions per BlockMix besides the arithmetic.  Counting method: every SASS instruction in a loop body except
    LOP3, SHF, IMAD and LEA, divided by the number of BlockMix bodies in the loop (its SHF count / 248: one BlockMix
    of rotate mask 0 has 248 funnel shifts)."""
import collections
import re
import shutil
import subprocess
from pathlib import Path

import pytest

SRC = Path(__file__).resolve().parent.parent / "go-spacemesh_b200" / "csrc" / "label_kernels.cu"
NVCC = shutil.which("nvcc") or ("/usr/local/cuda/bin/nvcc" if Path("/usr/local/cuda/bin/nvcc").exists() else None)
SHF_PER_BLOCKMIX = 248
MAX_OTHER_PER_BLOCKMIX = 40

pytestmark = pytest.mark.skipif(NVCC is None, reason="nvcc not found")


@pytest.fixture(scope="module")
def compiled(tmp_path_factory):
    cubin = tmp_path_factory.mktemp("sass") / "label_kernels.cubin"
    res = subprocess.run([NVCC, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-cubin", "-Xptxas", "-v",
                          "-o", str(cubin), str(SRC)], capture_output=True, text=True, cwd=SRC.parent)
    assert res.returncode == 0, res.stderr[-4000:]
    return cubin, res.stderr


def _sass(cubin, fn):
    out = subprocess.run([str(Path(NVCC).with_name("cuobjdump")), "-sass", "-fun", fn, str(cubin)],
                         capture_output=True, text=True, check=True).stdout
    ins = []
    for line in out.splitlines():
        m = re.match(r"\s*/\*([0-9a-f]{4,})\*/\s+(@!?U?P[T0-9]+\s+)?(.*?)\s*;", line)
        if m:
            ins.append((int(m.group(1), 16), bool(m.group(2)), m.group(3)))
    return ins


def _step_loops(ins):
    """(first, last) address of each loop closed by a conditional backward branch, other than the one-instruction
    waterfall loops ptxas builds around a UBLKCP (BRA.U.ANY)."""
    loops = []
    for a, pred, text in ins:
        t = re.match(r"BRA\s+0x([0-9a-f]+)", text)
        if pred and t and int(t.group(1), 16) < a:
            loops.append((int(t.group(1), 16), a))
    return loops


def test_phased_instances_fit_127_registers_without_spills(compiled):
    _, log = compiled
    parts = re.split(r"Compiling entry function '(\w+)'", log)
    blocks = [(fn, text) for fn, text in zip(parts[1::2], parts[2::2]) if "romix_phased_kernel" in fn]
    assert len(blocks) == 8
    for fn, text in blocks:
        regs = int(re.search(r"Used (\d+) registers", text).group(1))
        assert regs <= 127, (fn, regs)
        assert "0 bytes spill stores, 0 bytes spill loads" in text, (fn, text)


@pytest.mark.parametrize("mw", [0, 1])
@pytest.mark.parametrize("tpb", [64, 256, 512])
def test_phased_step_loops(compiled, mw, tpb):
    cubin, _ = compiled
    ins = _sass(cubin, f"_ZN8b200post19romix_phased_kernelILi{mw}ELi{tpb}EEEvNS_11RomixParamsE")
    loops = _step_loops(ins)
    kinds = collections.Counter()
    for lo, hi in loops:
        ops = collections.Counter(text.split()[0].split(".")[0] for a, _, text in ins if lo <= a <= hi)
        full = collections.Counter(text.split()[0] for a, _, text in ins if lo <= a <= hi)
        assert ops["SHFL"] == 0 and ops["WARPSYNC"] == 0 and ops["ENDCOLLECTIVE"] == 0, (hex(lo), ops)
        if ops["LDGSTS"]:
            kind = "mix"
        else:
            kind = "fill"
            assert ops["STG"] == 0, (hex(lo), ops)
            assert full["STS.128"] and ops["UBLKCP"] == full["STS.128"] // 8, (hex(lo), ops)   # one bulk store per tile
        kinds[kind] += 1
        if mw == 0:
            bodies = ops["SHF"] / SHF_PER_BLOCKMIX
            assert bodies in (1, 2), (hex(lo), ops)
            other = sum(n for op, n in ops.items() if op not in ("LOP3", "SHF", "IMAD", "LEA"))
            assert other / bodies <= MAX_OTHER_PER_BLOCKMIX, (hex(lo), other / bodies, ops)
    # paired and single-label fill and mix loops
    assert kinds == {"fill": 2, "mix": 2}, kinds
