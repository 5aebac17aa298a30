"""Rank -> GPU placement policies and the two mechanisms to apply them.

Capability parity with ``p2p/tile_mapping.sh:1-37`` of the reference, which computes a
``gpu.tile`` mask from ``PALS_LOCAL_RANKID`` by policy (compact | spread | compact_plan,
the last one asking ``./topology <rank>``) and exports it through ``ZE_AFFINITY_MASK`` (ZAM)
or ``ONEAPI_DEVICE_SELECTOR`` (ODS) before exec'ing the program.

H100 mapping of the two mechanisms:
  CVD  ``CUDA_VISIBLE_DEVICES=<gpu>``  — the process sees only its GPU (↔ ZAM)
  SET  ``HPCP_DEVICE=<gpu>``           — all GPUs stay visible, the program selects the
                                          ordinal with cudaSetDevice / torch.cuda.set_device (↔ ODS)
plus ``CUDA_DEVICE_ORDER=PCI_BUS_ID`` (↔ ``ZE_ENABLE_PCI_ID_DEVICE_ORDER=1``).

``python -m hpc_patterns_b200.parallel.tile_mapping <policy> <CVD|SET> cmd...`` is the
per-rank launcher; ``scripts/tile_mapping.sh`` is the same thing in bash.
"""
from __future__ import annotations

import json
import os
import shutil
import subprocess
import sys
from typing import List, Optional, Sequence

POLICIES = ("compact", "spread", "compact_plan")
MECHANISMS = ("CVD", "SET")
# The reference's spellings are accepted so its launch lines keep working (p2p/tile_mapping.sh:22-37):
# ZAM (ZE_AFFINITY_MASK: the process sees only its tile) and ODS (ONEAPI_DEVICE_SELECTOR: select by id).
MECHANISM_ALIASES = {"ZAM": "CVD", "ODS": "SET"}
_RANK_VARS = ("LOCAL_RANK", "OMPI_COMM_WORLD_LOCAL_RANK", "PALS_LOCAL_RANKID", "SLURM_LOCALID",
              "MPI_LOCALRANKID")


def local_rank(env=os.environ) -> int:
    for v in _RANK_VARS:
        if v in env:
            return int(env[v])
    raise RuntimeError("no local rank in the environment (looked for " + ", ".join(_RANK_VARS) + ")")


def flatten(planes: Sequence[Sequence[int]]) -> List[int]:
    return [g for p in planes for g in p]


def _spread(rank: int, n_devices: int, n_domains: int) -> int:
    """Round-robin over the domains (contiguous blocks of GPUs; the first n % d blocks hold one more), skipping a
    domain once it is exhausted — every GPU is used for any device count, and with equal blocks this is
    ``(r % d) * per + r // d``.  Identical in scripts/tile_mapping.sh and csrc/p2p/topology_core.cpp."""
    d = max(1, min(n_domains, n_devices))
    base, extra = divmod(n_devices, d)
    r = rank % n_devices
    seen = 0
    level = 0
    while True:
        for k in range(d):
            if level < base + (1 if k < extra else 0):
                if seen == r:
                    return k * base + min(k, extra) + level
                seen += 1
        level += 1


def device_for_rank(policy: str, rank: int, n_devices: int,
                    planes: Optional[Sequence[Sequence[int]]] = None, n_domains: int = 2) -> int:
    """Pure policy function (mirrors csrc/p2p/topology_core.cpp:device_for_rank)."""
    if n_devices <= 0:
        raise ValueError("no devices")
    if rank < 0:
        raise ValueError("negative rank")
    if policy == "compact":
        return rank % n_devices
    if policy == "spread":
        return _spread(rank, n_devices, n_domains)
    if policy == "compact_plan":
        flat = flatten(planes or [])
        if not flat:
            return rank % n_devices
        return flat[rank % len(flat)]
    raise ValueError(f"unknown policy {policy!r} (expected one of {POLICIES})")


def discover_planes(fake_spec: str = "") -> List[List[int]]:
    """Planes from the native topology code (NVML), or from a fake spec / $HPCP_FAKE_TOPOLOGY."""
    from .. import native

    info = json.loads(native().topology_discover(fake_spec or os.environ.get("HPCP_FAKE_TOPOLOGY", "")))
    return [list(p) for p in info["planes"]]


def count_devices(env=os.environ) -> int:
    if env.get("HPCP_NUM_DEVICES"):
        return int(env["HPCP_NUM_DEVICES"])
    exe = shutil.which("nvidia-smi")
    if exe:
        try:
            out = subprocess.run([exe, "-L"], capture_output=True, text=True, timeout=30).stdout
            n = sum(1 for line in out.splitlines() if line.startswith("GPU "))
            if n:
                return n
        except (OSError, subprocess.SubprocessError):
            pass
    raise RuntimeError("cannot count GPUs (set HPCP_NUM_DEVICES)")


def environment_for(policy: str, mechanism: str, rank: int, n_devices: int,
                    planes: Optional[Sequence[Sequence[int]]] = None) -> dict:
    """The variables the launcher exports for one rank."""
    mechanism = MECHANISM_ALIASES.get(mechanism, mechanism)
    if mechanism not in MECHANISMS:
        raise ValueError(f"WRONG AFFINITY MECHANISM {mechanism!r}: either CVD or SET")
    dev = device_for_rank(policy, rank, n_devices, planes)
    env = {"CUDA_DEVICE_ORDER": "PCI_BUS_ID"}
    if mechanism == "CVD":
        env["CUDA_VISIBLE_DEVICES"] = str(dev)
        env["HPCP_DEVICE"] = "0"
    else:
        env["HPCP_DEVICE"] = str(dev)
    return env


def selected_device(default: Optional[int] = None) -> int:
    """What a program launched under the wrapper should pass to ``torch.cuda.set_device``."""
    if "HPCP_DEVICE" in os.environ:
        return int(os.environ["HPCP_DEVICE"])
    if default is not None:
        return default
    return local_rank()


def main(argv: Optional[List[str]] = None) -> int:
    argv = list(sys.argv[1:] if argv is None else argv)
    if len(argv) < 3 or argv[0] not in POLICIES:
        print("usage: tile_mapping <compact|spread|compact_plan> <CVD|SET> cmd [args...]   (ZAM, ODS: aliases)", file=sys.stderr)
        return 2
    policy, mechanism, cmd = argv[0], argv[1], argv[2:]
    rank = local_rank()
    n = count_devices()
    planes = discover_planes() if policy == "compact_plan" else None
    env = dict(os.environ)
    env.update(environment_for(policy, mechanism, rank, n, planes))
    os.execvpe(cmd[0], cmd, env)
    return 0  # pragma: no cover


if __name__ == "__main__":
    raise SystemExit(main())
