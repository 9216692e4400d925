"""What the timing scripts under tools/ share: the card a number was measured on, a host clock around synchronised
calls, worker processes alternated over builds of the project with their outputs compared, the opaque-Module
wrapper, and the output convention (`--out DIR` writes DIR/<script>.json: the rows, every run and the card).

A script that compares builds runs each arm (a built tree of the project, with environment overrides such as
MPCB200_KERNEL) in worker processes of its own, because two builds share module names.  `alternate` starts
`script [args] --worker TREE OUT SAVE` once per arm and round, arm after arm; the worker calls `enter(TREE)` before it
imports the package and ends with `save(...)`."""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
LIB = os.path.join("mpc", "pytorch_b200", "libmpcb200.so")


def card(index=0):
    """Name, power limit (W) and maximum SM clock (MHz) of the card, read in the calling process."""
    import bench
    info = bench.device_info(index)
    mhz = None
    try:
        r = subprocess.run(["nvidia-smi", "-i", str(index), "--query-gpu=clocks.max.sm", "--format=csv,noheader,nounits"],
                           capture_output=True, text=True, timeout=30)
        mhz = int(r.stdout.strip())
    except (OSError, ValueError, subprocess.TimeoutExpired):
        pass
    return dict(name=info["name"], power_limit_w=info["power_limit_w"], sm_max_mhz=mhz)


def card_line(c):
    return f"card: {c['name']}, power limit {c['power_limit_w']} W, max SM clock {c['sm_max_mhz']} MHz"


def host_time(fn, reps):
    """Seconds of each of `reps` calls of `fn`, each followed by a device synchronise (a call returns before its
    kernels finish), and the last call's result."""
    torch.cuda.synchronize()
    ts, out = [], None
    for _ in range(reps):
        t0 = time.perf_counter()
        out = fn()
        torch.cuda.synchronize()
        ts.append(time.perf_counter() - t0)
    return ts, out


def add_arguments(ap, rounds=3):
    """The options of a script that alternates arms in worker processes."""
    ap.add_argument("--rounds", type=int, default=rounds, help="alternated worker processes per arm")
    ap.add_argument("--parent", default=None, help="another tree of the project, built, to compare against")
    ap.add_argument("--out", default=None, help="directory for <script>.json (default: print only)")
    ap.add_argument("--worker", nargs=3, metavar=("TREE", "OUT", "SAVE"), help=argparse.SUPPRESS)


def trees(parent):
    """{"this": this tree[, "parent": PARENT]}; PARENT must be a built tree of the project."""
    res = {"this": ROOT}
    if parent is not None:
        res["parent"] = os.path.abspath(parent)
        if not os.path.exists(os.path.join(res["parent"], LIB)):
            raise SystemExit(f"--parent {parent}: no {LIB} there; build that tree first")
    return res


def enter(tree):
    """In a worker: make `tree`'s package the one this process imports."""
    import bench  # noqa: F401  (importing bench puts this tree first on sys.path: do it before `tree` goes first)
    tree = os.path.abspath(tree)
    sys.path.insert(0, tree)
    import mpc.pytorch_b200 as pkg
    if not os.path.abspath(pkg.__file__).startswith(tree + os.sep):
        raise SystemExit(f"worker for {tree} imported {pkg.__file__}")


def save(out, times, info=None, outputs=None):
    """In a worker: write its timings ({row: [time, ...]}), JSON details per row and, if any, its outputs
    ({row: {name: tensor}})."""
    with open(out + ".json", "w") as fh:
        json.dump(dict(times=times, info=info or {}), fh)
    if outputs is not None:
        torch.save({r: {k: v.cpu() for k, v in d.items()} for r, d in outputs.items()}, out + ".pt")


def alternate(script, arms, rounds, args=()):
    """Runs `script *args --worker TREE OUT SAVE` for every arm (name -> (tree, environment overrides)) in turn,
    `rounds` times; SAVE is 1 in round 0 only.  Returns each arm's timings per row over all rounds, and its details
    and outputs from round 0."""
    times = {a: {} for a in arms}
    info, outs = {}, {}
    with tempfile.TemporaryDirectory() as tmp:
        for r in range(rounds):
            for i, (a, (tree, env)) in enumerate(arms.items()):
                out = os.path.join(tmp, f"{i}_{r}")
                subprocess.run([sys.executable, os.path.abspath(script), *args, "--worker", tree, out, str(int(r == 0))],
                               check=True, cwd=tmp, env={**os.environ, **env})
                with open(out + ".json") as fh:
                    res = json.load(fh)
                for row, ts in res["times"].items():
                    times[a].setdefault(row, []).extend(ts)
                if r == 0:
                    info[a] = res["info"]
                    outs[a] = torch.load(out + ".pt") if os.path.exists(out + ".pt") else {}
    return times, info, outs


def compare(mine, theirs):
    """Per output of one row (name -> tensor): whether the two are bitwise equal and, where not, the largest
    |difference|."""
    res = {}
    for k, a in mine.items():
        b = theirs.get(k)
        same = b is not None and a.shape == b.shape and a.dtype == b.dtype and torch.equal(a, b)
        res[f"{k}_bitwise"] = same
        if not same and b is not None and a.shape == b.shape:
            res[f"{k}_max_diff"] = float((a.double() - b.double()).abs().max())
    return res


class Opaque(torch.nn.Module):
    """A known system's physics without its mpcb200_kind: MPC treats it as an arbitrary Module (autograd
    linearisation, torch rollout), the route every system took before the kernels knew it."""

    def __init__(self, dx):
        super().__init__()
        self.dx = dx

    def forward(self, x, u):
        return self.dx(x, u)


def report(out, script, c, rows, runs, **extra):
    """Prints the card; with --out DIR, writes DIR/<script>.json: the card, the rows and every run."""
    print(card_line(c))
    if out is None:
        return
    os.makedirs(out, exist_ok=True)
    name = os.path.splitext(os.path.basename(script))[0]
    with open(os.path.join(out, name + ".json"), "w") as fh:
        json.dump(dict(card=c, torch=torch.__version__, rows=rows, runs=runs, **extra), fh, indent=1)
