"""Build libb200attn.so in-tree with nvcc for sm_90a (cross-compiles without a GPU).

The library is pure CUDA runtime + C ABI (``include/b200attn.h``): no torch headers, so a
rebuild takes seconds and the product .so travels to the GPU box with the snapshot.
"""

from __future__ import annotations

import hashlib
import os
import subprocess
import sys
from pathlib import Path
from typing import List

PKG_DIR = Path(__file__).resolve().parent
CSRC = PKG_DIR / "csrc"
INCLUDE = PKG_DIR.parent / "include"
LIB_PATH = PKG_DIR / "libb200attn.so"

SOURCES = [
    "capi.cu",
    "elementwise.cu",
    "activation.cu",
    "index_rows.cu",
    "metadata.cu",
    "attn_decode_bringup.cu",
    "attn_decode_tc.cu",
    "tma_host.cu",
    "attn_prefill_bringup.cu",
    "attn_prefill_tc.cu",
    "allreduce.cu",
]

NVCC_FLAGS = [
    "-gencode",
    "arch=compute_90a,code=sm_90a",
    "-O3",
    "-std=c++17",
    "-lineinfo",
    "--expt-relaxed-constexpr",
    "-Xcompiler",
    "-fPIC",
    "-Xcompiler",
    "-fvisibility=hidden",
    "-DB200_BUILDING=1",
]


def _flags() -> List[str]:
    """B200_BUILD_BRINGUP=1 adds the two cross-check kernels (cp.async decode, mma.sync prefill) that the
    parity tests can select with b200_set_option; the product build does not contain them."""
    extra = ["-DB200_BRINGUP_KERNELS=1"] if os.environ.get("B200_BUILD_BRINGUP", "0") not in ("", "0") else []
    return NVCC_FLAGS + extra


def _nvcc() -> str:
    cand = os.environ.get("NVCC") or "/usr/local/cuda/bin/nvcc"
    return cand if Path(cand).exists() else "nvcc"


def _digest(sources: List[Path]) -> str:
    h = hashlib.sha256()
    for f in sorted(list(CSRC.glob("*.cu*")) + list(INCLUDE.glob("*.h"))):
        h.update(f.name.encode())
        h.update(f.read_bytes())
    h.update(" ".join(_flags()).encode())
    h.update(" ".join(str(s.name) for s in sources).encode())
    return h.hexdigest()


def built_digest() -> str:
    """Digest the existing libb200attn.so carries ("B200DIGEST:<sha256>", also returned by
    ``b200_build_digest()``), "" if there is no library or it predates the marker.  The digest lives
    inside the binary, so a stale .so can never be mistaken for a current one (no side-car stamp
    file); it is read from the file bytes because dlopen-ing the old library here would pin it for
    the rest of the process."""
    if not LIB_PATH.exists():
        return ""
    import re

    m = re.search(rb"B200DIGEST:([0-9a-f]{64})", LIB_PATH.read_bytes())
    return m.group(1).decode() if m else ""


def build(force: bool = False, verbose: bool = False) -> Path:
    """Compile every .cu under csrc/ into libb200attn.so (skips when the library reports the digest
    of the current sources + flags)."""
    srcs = [CSRC / s for s in SOURCES]
    for s in srcs:
        if not s.exists():
            raise FileNotFoundError(s)
    digest = _digest(srcs)
    if not force and built_digest() == digest:
        return LIB_PATH
    objs = []
    procs = []
    build_dir = PKG_DIR / "build"
    build_dir.mkdir(exist_ok=True)
    for s in srcs:
        o = build_dir / (s.stem + ".o")
        cmd = [_nvcc(), *_flags(), "-I", str(INCLUDE), "-I", str(CSRC), "-c", str(s), "-o", str(o)]
        if s.name == "capi.cu":
            cmd.insert(1, f'-DB200_BUILD_DIGEST="B200DIGEST:{digest}"')
        if verbose:
            cmd.insert(1, "-Xptxas")
            cmd.insert(2, "-v")
        procs.append((s, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT)))
        objs.append(o)
    failed = False
    for s, pr in procs:
        out, _ = pr.communicate()
        text = out.decode(errors="replace")
        if pr.returncode != 0:
            failed = True
            sys.stderr.write(f"[b200 build] nvcc failed for {s.name}:\n{text}\n")
        elif verbose or text.strip():
            sys.stderr.write(f"[b200 build] {s.name}:\n{text}\n")
    if failed:
        raise RuntimeError("nvcc compilation failed (see stderr)")
    link = [
        _nvcc(),
        "-shared",
        "-gencode",
        "arch=compute_90a,code=sm_90a",
        "-o",
        str(LIB_PATH),
        *[str(o) for o in objs],
        "-cudart",
        "static",
    ]
    res = subprocess.run(link, stdout=subprocess.PIPE, stderr=subprocess.STDOUT)
    if res.returncode != 0:
        raise RuntimeError("link failed:\n" + res.stdout.decode(errors="replace"))
    return LIB_PATH


if __name__ == "__main__":
    p = build(force="--force" in sys.argv, verbose="-v" in sys.argv)
    print(p)
