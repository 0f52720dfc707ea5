"""Split the phased ROMix layer's time into its fill and mix phases at bench.py's batch.

The default library is timed against a scratch build of the same sources compiled with -DB200POST_PHASED_FILL_ONLY,
whose romix_phased_kernel stops after the fill loop (the labels it returns are wrong; only its time is used).  Fill time
is the fill-only call; mix time is the difference.  Each phase is set against its ceiling:
  - fill: the integer ALU pipe, N BlockMix steps x ALU_OPS_PER_BLOCKMIX lane-operations per label on 64 ALU lanes per SM
    at the sampled SM clock (bench.py's roofline, per phase);
  - mix: HBM, 128 * N bytes read per label at --hbm-tbps (3.07 TB/s is what tools/romix_traffic_probe.cu reaches for
    the phased traffic with no ChaCha on an H100 80GB HBM3 at 700 W).
A call also runs K1 and K3 (under 1 % of it); they are counted in the fill phase.

The libraries alternate, one process per timed run, so each run loads one library (B200POST_LIB).  Without
--fill-only-lib the scratch build is made in a temporary directory (a few minutes of nvcc).  Run on an H100 from the
repository root:
    python tools/romix_phase_split.py [--rounds 3] [--lib PATH] [--fill-only-lib PATH]
"""
import argparse
import json
import os
import shutil
import statistics
import subprocess
import sys
import tempfile
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
import bench  # noqa: E402  (ClockSampler, batch and N of the flagship workload)

ALU_OPS_PER_BLOCKMIX = 566    # ALU-pipe instructions per BlockMix, as in bench.py's integer roofline
ALU_LANES_PER_SM = 64


def build_fill_only(tmp: Path) -> Path:
    for d in ("go-spacemesh_b200/csrc", "include"):
        shutil.copytree(ROOT / d, tmp / d, ignore=shutil.ignore_patterns("build", "*.so"))
    subprocess.run(["make", "-C", str(tmp / "go-spacemesh_b200/csrc"), "-j8", "../libb200post.so",
                    "NVCC=nvcc -DB200POST_PHASED_FILL_ONLY"], check=True, capture_output=True, text=True)
    return tmp / "go-spacemesh_b200/libb200post.so"


def child(batch: int, calls: int) -> None:
    """One timed run in this process: warm-up call, then `calls` calls; prints the device ms of each."""
    from __graft_entry__ import load_package
    b2 = load_package()
    n = bench.N_SCRYPT
    commitment = b2.commitment(bytes(32), bytes(32))
    b2.labels_range(commitment, n, 0, batch, discard=True)
    ms = []
    for c in range(calls):
        b2.labels_range(commitment, n, (c + 1) * batch, batch, discard=True)
        ms.append(b2.last_call_ms())
    print(json.dumps({"call_ms": ms, "wave_slots": b2.wave_slots(n), "sm_count": b2.providers()[0]["sm_count"]}), flush=True)


def run(lib: Path, batch: int, calls: int) -> dict:
    env = dict(os.environ, B200POST_LIB=str(lib))
    out = subprocess.run([sys.executable, __file__, "--child", "--batch", str(batch), "--calls", str(calls)],
                         env=env, capture_output=True, text=True, check=True, cwd=ROOT).stdout
    return json.loads(out.strip().splitlines()[-1])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--calls", type=int, default=2, help="timed calls per run")
    ap.add_argument("--batch", type=int, default=bench.DEFAULT_BATCH)
    ap.add_argument("--lib", default=str(ROOT / "go-spacemesh_b200/libb200post.so"))
    ap.add_argument("--fill-only-lib", help="a library built with -DB200POST_PHASED_FILL_ONLY (default: build one)")
    ap.add_argument("--hbm-tbps", type=float, default=3.07)
    ap.add_argument("--child", action="store_true", help=argparse.SUPPRESS)
    args = ap.parse_args()
    if args.child:
        return child(args.batch, args.calls)
    with tempfile.TemporaryDirectory() as td:
        fill_lib = Path(args.fill_only_lib) if args.fill_only_lib else build_fill_only(Path(td))
        libs = {"full": Path(args.lib), "fill": fill_lib}
        ms = {"full": [], "fill": []}
        sms = 0
        sampler = bench.ClockSampler(0)
        sampler.start()
        for r in range(args.rounds):
            for name, lib in libs.items():
                res = run(lib, args.batch, args.calls)
                ms[name] += res["call_ms"]
                sms = res["sm_count"]
                print(json.dumps({"lib": name, "round": r, **res}), flush=True)
        clocks = sampler.stop()
    q = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip()
    n, batch = bench.N_SCRYPT, args.batch
    full, fill = statistics.median(ms["full"]) / 1e3, statistics.median(ms["fill"]) / 1e3
    mix = full - fill
    clock_mhz = clocks.get("sm_mhz")
    alu_s = batch * n * ALU_OPS_PER_BLOCKMIX / (sms * ALU_LANES_PER_SM * clock_mhz * 1e6) if clock_mhz else None
    hbm_s = batch * 128 * n / (args.hbm_tbps * 1e12)
    print(json.dumps({
        "card": q, "batch": batch, "N": n, "clocks": clocks,
        "spread": {k: (max(v) - min(v)) / min(v) for k, v in ms.items()},
        "full_s": full, "fill_s": fill, "mix_s": mix, "labels_per_s": batch / full,
        "fill_alu_ceiling_s": alu_s, "fill_over_alu_ceiling": alu_s / fill if alu_s else None,
        "mix_hbm_ceiling_s": hbm_s, "mix_over_hbm_ceiling": hbm_s / mix,
        "mix_alu_ceiling_s": alu_s,
    }), flush=True)


if __name__ == "__main__":
    main()
