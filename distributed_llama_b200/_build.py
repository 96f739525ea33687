"""In-tree builder for the two native libraries.

* ``_host``  – pybind11 module (g++ only): formats, codecs, slicers, tokenizer, sampler.
* ``_cuda``  – plain C-ABI shared library (nvcc, sm_90a only): kernels, engine runtime, peer-memory comm.
  Loaded through ctypes so the kernels carry no torch/pybind dependency and compile in seconds.

Artifacts are written next to this file (git-ignored).
A source hash is stored beside each artifact so stale builds are rebuilt and fresh ones are reused.
"""
from __future__ import annotations

import hashlib
import os
import shutil
import subprocess
import sys
import sysconfig
import threading
from pathlib import Path

PKG_DIR = Path(__file__).resolve().parent
REPO_DIR = PKG_DIR.parent
CSRC = REPO_DIR / "csrc"
_lock = threading.Lock()

NVCC_ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]


def _hash_sources(files, extra: str = "") -> str:
    h = hashlib.sha256(extra.encode())
    for f in sorted(files):
        h.update(str(f.name).encode())
        h.update(f.read_bytes())
    return h.hexdigest()


def _run(cmd, cwd=None):
    proc = subprocess.run(cmd, cwd=cwd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if proc.returncode != 0:
        raise RuntimeError("build command failed:\n  " + " ".join(map(str, cmd)) + "\n" + proc.stdout)
    return proc.stdout


def host_lib_path() -> Path:
    return PKG_DIR / ("_host" + sysconfig.get_config_var("EXT_SUFFIX"))


def cuda_lib_path() -> Path:
    return PKG_DIR / "_cuda.so"


def build_host(force: bool = False, verbose: bool = False) -> Path:
    src_dir = CSRC / "host"
    sources = sorted(src_dir.glob("*.cpp"))
    headers = sorted(src_dir.glob("*.hpp"))
    out = host_lib_path()
    stamp = out.with_suffix(out.suffix + ".hash")
    flags = ["-O2", "-std=c++17", "-fPIC", "-shared", "-fvisibility=hidden", "-Wall", "-Wno-sign-compare"]
    if os.environ.get("DLLAMA_DEBUG") == "1":
        # reference: `make DEBUG=1` => -g -fsanitize=address (Makefile:8-12). Run python with LD_PRELOAD=$(g++ -print-file-name=libasan.so).
        flags = ["-O1", "-g", "-fsanitize=address", "-fno-omit-frame-pointer"] + flags[1:]
    digest = _hash_sources(sources + headers, " ".join(flags))
    with _lock:
        if not force and out.exists() and stamp.exists() and stamp.read_text() == digest:
            return out
        import pybind11

        inc = ["-I" + sysconfig.get_paths()["include"], "-I" + pybind11.get_include()]
        tmp = out.with_suffix(".tmp.so")
        cmd = ["g++", *flags, *inc, *map(str, sources), "-o", str(tmp)]
        log = _run(cmd)
        if verbose and log:
            print(log)
        os.replace(tmp, out)
        stamp.write_text(digest)
    return out


def nvcc_path() -> str:
    for cand in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and os.path.exists(cand):
            return cand
    raise RuntimeError("nvcc not found")


def build_cuda(force: bool = False, verbose: bool = False) -> Path:
    src_dir = CSRC / "cuda"
    sources = sorted(src_dir.glob("*.cu"))
    headers = sorted(src_dir.glob("*.cuh")) + sorted(src_dir.glob("*.h"))
    out = cuda_lib_path()
    stamp = out.with_suffix(".so.hash")
    flags = [*NVCC_ARCH, "-O3", "-std=c++17", "-lineinfo", "--use_fast_math", "-Xcompiler", "-fPIC",
             "-Xcompiler", "-fvisibility=hidden", "--expt-relaxed-constexpr", "-Xptxas", "-v"]
    if os.environ.get("DLLAMA_DEBUG") == "1":
        flags = [f for f in flags if f not in ("-O3", "--use_fast_math")] + ["-O1", "-g"]   # device code stays optimised; tools/sanitize.sh
    digest = _hash_sources(sources + headers, " ".join(flags))
    with _lock:
        if not force and out.exists() and stamp.exists() and stamp.read_text() == digest:
            return out
        nvcc = nvcc_path()
        obj_dir = REPO_DIR / "build" / "cuda"
        obj_dir.mkdir(parents=True, exist_ok=True)
        objs = []
        procs = []
        for s in sources:
            o = obj_dir / (s.stem + ".o")
            objs.append(o)
            ostamp = o.with_suffix(".o.hash")
            odigest = _hash_sources([s] + headers, " ".join(flags))
            if not force and o.exists() and ostamp.exists() and ostamp.read_text() == odigest:
                continue
            cmd = [nvcc, *flags, "-c", str(s), "-o", str(o)]
            procs.append((s, o, ostamp, odigest, cmd,
                          subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
        logs = []
        for s, o, ostamp, odigest, cmd, p in procs:
            text, _ = p.communicate()
            logs.append(f"== {s.name}\n{text}")
            if p.returncode != 0:
                raise RuntimeError("nvcc failed:\n  " + " ".join(cmd) + "\n" + text)
            ostamp.write_text(odigest)
        (obj_dir / "ptxas.log").write_text("\n".join(logs))
        if verbose:
            print("\n".join(logs))
        tmp = out.with_suffix(".tmp.so")
        _run([nvcc, *NVCC_ARCH, "-shared", "-o", str(tmp), *map(str, objs)])
        os.replace(tmp, out)
        stamp.write_text(digest)
    return out


NATIVE_BINARIES = {"dllama-native": "dllama_main.cpp", "dllama-api-native": "dllama_api_main.cpp"}


def native_bin_path(name: str = "dllama-native") -> Path:
    return PKG_DIR / name


def build_native(force: bool = False, verbose: bool = False):
    """The Python-free front ends: csrc/app (CLI, API server, engine driver) + csrc/host (formats, tokenizer, sampler) linked
    against _cuda.so and the CUDA runtime. Reference counterparts: the `dllama` / `dllama-api` make targets (Makefile:40-66)."""
    cuda_so = build_cuda(force, verbose)
    app = CSRC / "app"
    common = [app / "native_engine.cpp", app / "api_server.cpp"] + [CSRC / "host" / n for n in ("quants.cpp", "model_format.cpp", "text.cpp")]
    headers = sorted(app.glob("*.hpp")) + sorted((CSRC / "host").glob("*.hpp")) + [CSRC / "cuda" / "engine_api.h"]
    cuda_home = Path(nvcc_path()).resolve().parent.parent
    flags = ["-O2", "-std=c++17", "-Wall", "-Wno-sign-compare", f"-I{cuda_home}/include"]
    link = [f"-L{PKG_DIR}", "-l:_cuda.so", f"-L{cuda_home}/lib64", "-lcudart", "-lpthread", "-Wl,-rpath,$ORIGIN", f"-Wl,-rpath,{cuda_home}/lib64"]
    outs = []
    for name, main_src in NATIVE_BINARIES.items():
        sources = [app / main_src] + common
        out = native_bin_path(name)
        stamp = out.with_suffix(".hash")
        digest = _hash_sources(sources + headers + [cuda_so.with_suffix(".so.hash")], " ".join(flags + link))
        with _lock:
            if force or not out.exists() or not stamp.exists() or stamp.read_text() != digest:
                tmp = out.with_suffix(".tmp")
                log = _run(["g++", *flags, *map(str, sources), *link, "-o", str(tmp)])
                if verbose and log:
                    print(log)
                os.replace(tmp, out)
                stamp.write_text(digest)
        outs.append(out)
    return outs


def build_all(force: bool = False, verbose: bool = False):
    return [build_host(force, verbose), build_cuda(force, verbose), *build_native(force, verbose)]


if __name__ == "__main__":
    force = "--force" in sys.argv
    for path in build_all(force=force, verbose="-v" in sys.argv):
        print(path)
