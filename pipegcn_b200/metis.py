"""`--partition-method metis` (PipeGCN/helper/parser.py:39-41, helper/utils.py:143-144).

The reference partitions through DGL, which calls METIS `PartGraphKway` with the `cut` or `vol` objective.  DGL is
absent; METIS itself ships as a static library inside the CUDA toolkit (`libmetis_static.a`, idx_t = int64,
real_t = float -- SURVEY.md §0.5).  It is wrapped into a small shared object once (gcc, no sources copied) and called
through ctypes on the symmetric adjacency without self loops.  Host-side set-up code, not part of the timed path.
"""
from __future__ import annotations

import ctypes as C
import subprocess
from pathlib import Path

import numpy as np
import torch

_HERE = Path(__file__).resolve().parent
_LIB = _HERE / "libpg_metis.so"
_ARCHIVES = ["/usr/local/cuda/targets/x86_64-linux/lib/libmetis_static.a", "/usr/local/cuda/lib64/libmetis_static.a"]

METIS_NOPTIONS = 40
OPT_OBJTYPE, OPT_SEED, OPT_NUMBERING = 1, 8, 17


def build(force: bool = False) -> Path:
    if _LIB.exists() and not force:
        return _LIB
    archive = next((a for a in _ARCHIVES if Path(a).exists()), None)
    if archive is None:
        raise RuntimeError("libmetis_static.a not found in the CUDA toolkit; use --partition-method random")
    # several ranks may get here at once (spawned processes): link into a private file, publish it atomically
    import os
    tmp = _LIB.with_suffix(f".so.tmp{os.getpid()}")
    subprocess.run(["gcc", "-shared", "-fPIC", "-o", str(tmp), "-Wl,--whole-archive", archive,
                    "-Wl,--no-whole-archive", "-lm"], check=True)
    os.replace(tmp, _LIB)
    return _LIB


_lib = None


def _metis():
    global _lib
    if _lib is None:
        _lib = C.CDLL(str(build()))
        _lib.METIS_SetDefaultOptions.argtypes = [C.c_void_p]
        _lib.METIS_PartGraphKway.argtypes = [C.c_void_p] * 13
        _lib.METIS_PartGraphKway.restype = C.c_int
    return _lib


def metis_partition(g, n_parts: int, objtype: str = "vol", seed: int = 0) -> torch.Tensor:
    """Node -> part assignment of `g` (a GlobalGraph) with METIS k-way, objective `cut` or `vol`."""
    n = g.n_nodes
    if n_parts <= 1:
        return torch.zeros(n, dtype=torch.int64, device=g.src.device)
    src, dst = g.src.cpu(), g.dst.cpu()
    keep = src != dst
    src, dst = src[keep], dst[keep]
    key = torch.unique(torch.cat([src * n + dst, dst * n + src]))        # symmetric, deduplicated
    rows, cols = (key // n).numpy(), (key % n).numpy()
    xadj = np.zeros(n + 1, dtype=np.int64)
    np.cumsum(np.bincount(rows, minlength=n), out=xadj[1:])
    adjncy = np.ascontiguousarray(cols, dtype=np.int64)
    lib = _metis()
    options = np.zeros(METIS_NOPTIONS, dtype=np.int64)
    lib.METIS_SetDefaultOptions(options.ctypes.data)
    options[OPT_OBJTYPE] = 1 if objtype == "vol" else 0
    options[OPT_SEED] = seed
    options[OPT_NUMBERING] = 0
    nvtxs, ncon, nparts, objval = (np.array([v], dtype=np.int64) for v in (n, 1, n_parts, 0))
    part = np.zeros(n, dtype=np.int64)
    rc = lib.METIS_PartGraphKway(nvtxs.ctypes.data, ncon.ctypes.data, xadj.ctypes.data, adjncy.ctypes.data,
                                 None, None, None, nparts.ctypes.data, None, None, options.ctypes.data,
                                 objval.ctypes.data, part.ctypes.data)
    if rc != 1:
        raise RuntimeError(f"METIS_PartGraphKway failed ({rc})")
    return torch.from_numpy(part).to(g.src.device)
