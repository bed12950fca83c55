"""Two (or more) builds of the library alternated on one card through BMB200_LIB: C3 three times and C2 / C5 twice per build with
`bench.py --no-e2e --no-cpu --no-parity` (default steps), then `scripts/bench_run_lists.py` (AND = {1, 2} and {1, 601}) per build.
The first bench run of each workload per build also writes `--dump-outputs` into a temporary directory; the dumps of every build
are compared byte for byte with those of the first.  Prints the card (name, power limit, max SM clock), min-max ms per step per
build, and C3's streamed bytes (from bench_run_lists, AND = {1, 2}) per second against the read ceiling of
scripts/microbench_read.cu (3191 GB/s on an H100 80GB HBM3 SXM at 700 W).
python scripts/bench_pipe_stages.py BASE_LIB [LIB ...]   (from the repository root, on an H100; LIB defaults to the tree's library)
BASE_LIB is e.g. the parent commit's libbmb200.so, compiled with build()'s nvcc line into an untracked path."""
import argparse
import filecmp
import json
import os
import subprocess
import sys
import tempfile
from pathlib import Path

ROOT = Path(__file__).resolve().parents[1]
READ_CEILING_GBS = 3191.0

ap = argparse.ArgumentParser()
ap.add_argument("libs", nargs="+", help="libbmb200.so builds; the first is the base the others are compared with")
ap.add_argument("--c3-runs", type=int, default=3)
ap.add_argument("--c2-runs", type=int, default=2)
ap.add_argument("--c5-runs", type=int, default=2)
ap.add_argument("--no-run-lists", action="store_true", help="skip bench_run_lists.py")
args = ap.parse_args()
libs = [str(Path(p).resolve()) for p in args.libs]
if len(libs) == 1:
    libs.append(str(ROOT / "bitmagic_b200" / "libbmb200.so"))
for p in libs:
    if not Path(p).is_file():
        sys.exit("no such library: " + p)

card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                      capture_output=True, text=True, check=True).stdout.strip()
print(json.dumps({"card": card, "libs": libs}), flush=True)


def run(lib, cmd):
    env = dict(os.environ, BMB200_LIB=lib)
    out = subprocess.run([sys.executable] + cmd, cwd=ROOT, env=env, capture_output=True, text=True)
    if out.returncode != 0:
        sys.exit("%s failed with %s:\n%s" % (" ".join(cmd), lib, out.stdout[-2000:] + out.stderr[-4000:]))
    return [json.loads(l) for l in out.stdout.splitlines() if l.startswith("{")]


tmp = Path(tempfile.mkdtemp(prefix="bench_pipe_stages_"))
ms = {}
for wl, reps in (("c3", args.c3_runs), ("c2", args.c2_runs), ("c5", args.c5_runs)):
    for rep in range(reps):
        for i, lib in enumerate(libs):
            cmd = ["bench.py", "--workload", wl, "--no-e2e", "--no-cpu", "--no-parity"]
            if rep == 0:
                cmd += ["--dump-outputs", str(tmp / str(i) / wl)]
            line = [l for l in run(lib, cmd) if "ms_per_step" in l][-1]
            ms.setdefault(wl, {}).setdefault(i, []).append(line["ms_per_step"])
            print(json.dumps({"workload": wl, "lib": i, "ms_per_step": line["ms_per_step"]}), flush=True)

same = {}
for wl in ms:
    for i in range(1, len(libs)):
        a, b = tmp / "0" / wl, tmp / str(i) / wl
        names = sorted(p.name for p in a.iterdir())
        match, mismatch, errors = filecmp.cmpfiles(a, b, names, shallow=False)
        same["%s_lib%d" % (wl, i)] = bool(names) and not mismatch and not errors and sorted(p.name for p in b.iterdir()) == names

streamed = {}
if not args.no_run_lists:
    for i, lib in enumerate(libs):
        for l in run(lib, ["scripts/bench_run_lists.py"]):
            print(json.dumps({"lib": i, "bench_run_lists": l}), flush=True)
            if l.get("and_group") == [1, 2]:
                streamed[i] = l.get("streamed_bytes", l["streamed_bytes_mode1"])   # what the default path streams

summary = {"card": card, "dumps_identical": same}
for wl in ms:
    for i, v in ms[wl].items():
        row = {"min": min(v), "max": max(v)}
        if wl == "c3" and i in streamed:
            gbs = streamed[i] / (min(v) * 1e-3) / 1e9
            row.update(streamed_gb=round(streamed[i] / 1e9, 3), streamed_gbs=round(gbs, 1), of_read_ceiling=round(gbs / READ_CEILING_GBS, 3))
        summary["%s_lib%d" % (wl, i)] = row
print(json.dumps(summary), flush=True)
