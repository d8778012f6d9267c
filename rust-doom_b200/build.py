"""Build recipe for libb2d.so: nvcc, sm_90a only, in-tree output (rust-doom_b200/libb2d.so).

`python -m rust_doom_b200.build` (or __graft_entry__.build()).  nvcc cross-compiles without a GPU.
"""
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
OUT = os.path.join(HERE, "libb2d.so")
SOURCES = ["b2d_api.cu", "b2d_kernels.cu", "b2d_sharded.cu", "b2d_wad.cpp", "b2d_scene.cpp"]
HEADERS = ["b2d_cli.cpp", "b2d_math.cuh", "b2d_kernels.cuh", "b2d_internal.hpp", "b2d_scene.hpp", "b2d_wad.hpp", "../../include/b2d.h"]

NVCC_FLAGS = ["-O3", "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo",
              "-Xcompiler", "-fPIC,-Wall,-Wextra,-Wno-unused-parameter", "-shared",
              "-Xptxas", "-v" if os.environ.get("B2D_PTXAS_V") else "-warn-spills", "-ldl"]


INFO = os.path.join(HERE, "libb2d.build.json")


def source_digest() -> str:
    """sha256 over the library's sources and headers (what a build is a function of, besides the compiler)."""
    import hashlib
    h = hashlib.sha256()
    for f in sorted(set(SOURCES + HEADERS + ["b2d_thing_table.inc", "b2d_anim_table.inc"])):
        p = os.path.join(CSRC, f)
        if os.path.exists(p):
            h.update(f.encode())
            with open(p, "rb") as fh:
                h.update(fh.read())
    return h.hexdigest()[:16]


def build_info() -> dict:
    """What produced the in-tree libb2d.so (written next to it by build()); bench.py puts it on its JSON line together with
    whether the sources still match, so a run shows which build of which sources it measured."""
    import json
    try:
        with open(INFO) as f:
            info = json.load(f)
    except Exception:  # noqa: BLE001
        info = {"recorded": False}
    info["sources_now"] = source_digest()
    info["sources_match"] = info.get("sources") == info["sources_now"]
    return info


def needs_build() -> bool:
    if not os.path.exists(OUT) or not os.path.exists(os.path.join(HERE, "b2d")):
        return True
    t = os.path.getmtime(OUT)
    if any(os.path.getmtime(os.path.join(CSRC, f)) > t for f in SOURCES + HEADERS):
        return True
    # mtimes do not survive every copy (a snapshot to another box): the recorded source digest decides
    info = build_info()
    return bool(info.get("recorded")) and not info["sources_match"]


def build(force: bool = False, verbose: bool = False) -> str:
    if not force and not needs_build():
        return OUT
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    cmd = [nvcc] + NVCC_FLAGS + ["-o", OUT] + [os.path.join(CSRC, s) for s in SOURCES]
    if verbose:
        print(" ".join(cmd))
    subprocess.check_call(cmd)
    build_cli(verbose)
    import json
    import socket
    import time
    try:
        ver = subprocess.run([nvcc, "--version"], capture_output=True, text=True).stdout.strip().splitlines()[-2:]
    except Exception:  # noqa: BLE001
        ver = []
    with open(INFO, "w") as f:
        json.dump({"recorded": True, "sources": source_digest(), "nvcc": " | ".join(ver), "flags": " ".join(NVCC_FLAGS),
                   "host": socket.gethostname(), "when": time.strftime("%Y-%m-%dT%H:%M:%SZ", time.gmtime())}, f, indent=1)
    return OUT


CLI_OUT = os.path.join(HERE, "b2d")


def build_cli(verbose: bool = False) -> str:
    """The compiled front end on the C ABI (csrc/b2d_cli.cpp): plain g++, links libb2d.so, rpath = its directory."""
    cmd = [os.environ.get("CXX", "g++"), "-O2", "-std=c++17", "-Wall", "-Wextra", "-o", CLI_OUT,
           os.path.join(CSRC, "b2d_cli.cpp"), "-L" + HERE, "-lb2d", "-Wl,-rpath,$ORIGIN"]
    if verbose:
        print(" ".join(cmd))
    subprocess.check_call(cmd)
    return CLI_OUT


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose=True))
