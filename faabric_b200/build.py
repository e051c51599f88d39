"""In-tree native build of libfaabric_b200.so (and the C++ binaries).

Every ``.cu`` under ``csrc/kernels`` is compiled by nvcc for sm_90a ONLY
(``-gencode arch=compute_90a,code=sm_90a -lineinfo``); host C++ is compiled
with g++ -std=c++20.  Objects are cached under ``build/obj`` keyed by a hash of
(source, headers mtime, flags) so incremental rebuilds are fast.  The result is
written to ``faabric_b200/lib/libfaabric_b200.so`` so it travels with the tree.

CLI:  python -m faabric_b200.build [--force] [--bins] [--jobs N]
"""

from __future__ import annotations

import concurrent.futures as cf
import hashlib
import os
import shutil
import subprocess
import sys
import time
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
CSRC = ROOT / "csrc"
BUILD = ROOT / "build"
OBJ = BUILD / "obj"
LIBDIR = ROOT / "faabric_b200" / "lib"
LIB = LIBDIR / "libfaabric_b200.so"
BINDIR = BUILD / "bin"

CUDA_HOME = Path(os.environ.get("CUDA_HOME", "/usr/local/cuda"))
NVCC = str(CUDA_HOME / "bin" / "nvcc")

ARCH_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a"]
NVCC_FLAGS = [
    "-std=c++17",
    "-O3",
    "-lineinfo",
    "-Xcompiler",
    "-fPIC",
    "--expt-relaxed-constexpr",
    "-Xptxas",
    "-v",
] + ARCH_FLAGS
CXX = os.environ.get("CXX", "g++")
CXX_FLAGS = [
    "-std=c++20",
    "-O2",
    "-g",
    "-fPIC",
    "-fno-omit-frame-pointer",
    "-Wall",
    "-Wno-unused-function",
    "-pthread",
]
# FAABRIC_B200_SANITISE=address|thread|undefined instruments the HOST code
_SAN = os.environ.get("FAABRIC_B200_SANITISE", "")
if _SAN:
    CXX_FLAGS += [f"-fsanitize={_SAN}", "-O1"]
# FAABRIC_B200_COVERAGE=1: gcov instrumentation of the host code (the
# reference's FAABRIC_CODE_COVERAGE option); see `cli coverage`
_COV = os.environ.get("FAABRIC_B200_COVERAGE", "") not in ("", "0")
if _COV:
    CXX_FLAGS = [f for f in CXX_FLAGS if f != "-O2"] + ["--coverage", "-O0"]
INCLUDES = [
    f"-I{CSRC / 'include'}",
    f"-I{CSRC / 'kernels'}",
    f"-I{CSRC / 'src'}",
    f"-I{CUDA_HOME / 'include'}",
]


_STDCXX_FLAGS: list[str] | None = None


def _stdcxx_link_flags() -> list[str]:
    """Make sure libstdc++ is linked as the SHARED system library.

    Some toolchain wrappers (e.g. a ``$CXX`` whose private lib dir only has a
    usable ``libstdc++.a``) silently link libstdc++ statically.  A second copy
    of libstdc++ inside libfaabric_b200.so, loaded into a Python process next
    to torch's libstdc++.so.6, mixes the two runtimes (locale facets!) and
    crashes in iostream code.  If the probe link does not depend on
    libstdc++.so, point the linker at the directory that holds the system one.
    """
    global _STDCXX_FLAGS
    if _STDCXX_FLAGS is not None:
        return _STDCXX_FLAGS
    flags: list[str] = []
    try:
        probe_dir = BUILD / "probe"
        probe_dir.mkdir(parents=True, exist_ok=True)
        src = probe_dir / "p.cpp"
        src.write_text("#include <string>\nstd::string fb_probe(){return std::string(40, 'x');}\n")
        out = probe_dir / "libp.so"

        def links_shared(extra):
            r = subprocess.run([CXX, "-shared", "-fPIC", str(src), "-o", str(out)] + extra, capture_output=True, text=True)
            if r.returncode != 0:
                return False
            d = subprocess.run(["readelf", "-d", str(out)], capture_output=True, text=True).stdout
            return "libstdc++.so" in d

        if not links_shared([]):
            for cand in ("g++", "/usr/bin/g++", "c++"):
                exe = shutil.which(cand)
                if not exe:
                    continue
                f = subprocess.run([exe, "-print-file-name=libstdc++.so"], capture_output=True, text=True).stdout.strip()
                if f and os.path.isabs(f) and os.path.exists(f):
                    extra = [f"-L{os.path.dirname(f)}"]
                    if links_shared(extra):
                        flags = extra
                        break
    except OSError:
        pass
    _STDCXX_FLAGS = flags
    return flags


def _stamp_of(paths) -> str:
    h = hashlib.sha1()
    for p in sorted(paths):
        st = p.stat()
        h.update(f"{p}:{st.st_mtime_ns}:{st.st_size}".encode())
    return h.hexdigest()


def _headers_stamp() -> dict:
    """Two stamps: kernels (.cu) only depend on csrc/kernels + the device ABI
    headers, host code depends on every header."""
    kernel_hdrs = list((CSRC / "kernels").glob("*.cuh")) + list((CSRC / "kernels").glob("*.h")) + list(
        (CSRC / "include" / "faabric" / "device").glob("*.h")
    )
    all_hdrs = []
    for pat in ("**/*.h", "**/*.cuh", "**/*.hpp"):
        all_hdrs += list(CSRC.glob(pat))
    return {"cu": _stamp_of(kernel_hdrs), "cpp": _stamp_of(all_hdrs)}


def _sources():
    cu = sorted((CSRC / "kernels").glob("*.cu"))
    cpp = sorted((CSRC / "src").glob("**/*.cpp")) + sorted(
        (CSRC / "capi").glob("*.cpp")
    )
    return cu, cpp


def _obj_for(src: Path) -> Path:
    rel = src.relative_to(CSRC)
    return OBJ / (str(rel).replace("/", "__") + ".o")


def _compile(src: Path, stamp, force: bool, extra_defs=()) -> tuple[Path, float, str]:
    obj = _obj_for(src)
    is_cu = src.suffix == ".cu"
    cmd = (
        [NVCC] + NVCC_FLAGS + INCLUDES + list(extra_defs) + ["-c", str(src), "-o", str(obj)]
        if is_cu
        else [CXX] + CXX_FLAGS + INCLUDES + list(extra_defs) + ["-c", str(src), "-o", str(obj)]
    )
    stamp_s = stamp["cu" if is_cu else "cpp"] if isinstance(stamp, dict) else stamp
    key = hashlib.sha1(
        (" ".join(cmd) + stamp_s + str(src.stat().st_mtime_ns)).encode()
    ).hexdigest()
    keyfile = obj.with_suffix(".key")
    if (
        not force
        and obj.exists()
        and keyfile.exists()
        and keyfile.read_text() == key
    ):
        return obj, 0.0, ""
    t0 = time.time()
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError(f"compile failed: {' '.join(cmd)}\n{r.stdout}\n{r.stderr}")
    keyfile.write_text(key)
    log = r.stderr if is_cu else ""
    return obj, time.time() - t0, log


def build(force: bool = False, bins: bool = True, jobs: int | None = None, verbose: bool = True) -> Path:
    if shutil.which(NVCC) is None and not Path(NVCC).exists():
        raise RuntimeError(f"nvcc not found at {NVCC}")
    OBJ.mkdir(parents=True, exist_ok=True)
    LIBDIR.mkdir(parents=True, exist_ok=True)
    BINDIR.mkdir(parents=True, exist_ok=True)
    stamp = _headers_stamp()
    cu, cpp = _sources()
    jobs = jobs or max(2, (os.cpu_count() or 4))
    t0 = time.time()
    objs: list[Path] = []
    ptxas_log: list[str] = []
    rebuilt = 0
    # longest compiles first
    order = sorted(cu, key=lambda p: -p.stat().st_size) + cpp
    with cf.ThreadPoolExecutor(max_workers=jobs) as ex:
        futs = {ex.submit(_compile, s, stamp, force): s for s in order}
        for f in cf.as_completed(futs):
            obj, dt, log = f.result()
            objs.append(obj)
            if dt > 0:
                rebuilt += 1
                if verbose:
                    print(f"  [{dt:5.1f}s] {futs[f].relative_to(CSRC)}", flush=True)
            if log:
                ptxas_log.append(f"## {futs[f].name}\n{log}")
    objs.sort()
    need_link = rebuilt > 0 or not LIB.exists() or force
    if need_link:
        cmd = (
            [CXX, "-shared", "-o", str(LIB)]
            + _stdcxx_link_flags()
            + [str(o) for o in objs]
            + [
                f"-L{CUDA_HOME / 'lib64'}",
                "-lcudart_static",
                "-ldl",
                "-lrt",
                "-lpthread",
                "-Wl,--no-undefined",
                "-Wl,--export-dynamic",
            ]
            + ([f"-fsanitize={_SAN}"] if _SAN else [])
            + (["--coverage"] if _COV else [])
        )
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError(f"link failed:\n{r.stdout}\n{r.stderr}")
    if ptxas_log:
        (BUILD / "ptxas_v.log").write_text("\n".join(ptxas_log))
    if bins:
        _build_bins(stamp, force or need_link, verbose)
    if verbose:
        print(
            f"faabric_b200: built {LIB} ({rebuilt} objects rebuilt, "
            f"{time.time() - t0:.1f}s)",
            flush=True,
        )
    return LIB


def _build_bins(stamp, relink: bool, verbose: bool) -> None:
    """C++ executables: test runner, planner_server, examples, benchmarks."""
    for sub in ("bin", "tests"):
        d = CSRC / sub
        if not d.exists():
            continue
        groups: dict[str, list[Path]] = {}
        for src in sorted(d.glob("*.cpp")):
            # tests/*.cpp all link into one runner; bin/*.cpp are one binary each
            name = "faabric_tests" if sub == "tests" else src.stem
            groups.setdefault(name, []).append(src)
        for name, srcs in groups.items():
            out = BINDIR / name
            objs = []
            rebuilt = False
            with cf.ThreadPoolExecutor(max_workers=os.cpu_count() or 4) as ex:
                for obj, dt, _ in ex.map(lambda s: _compile(s, stamp, False), srcs):
                    objs.append(obj)
                    rebuilt = rebuilt or dt > 0
            if rebuilt or relink or not out.exists():
                cmd = (
                    [CXX, "-o", str(out)]
                    + _stdcxx_link_flags()
                    + [str(o) for o in objs]
                    + [
                        f"-L{LIBDIR}",
                        "-lfaabric_b200",
                        f"-Wl,-rpath,{LIBDIR}",
                        "-Wl,-rpath,$ORIGIN/../../faabric_b200/lib",
                        # the GPU tests allocate device buffers themselves
                        f"-L{CUDA_HOME / 'lib64'}",
                        "-lcudart_static",
                        "-lrt",
                        "-lpthread",
                        "-ldl",
                    ]
                    + ([f"-fsanitize={_SAN}"] if _SAN else [])
                    + (["--coverage"] if _COV else [])
                )
                r = subprocess.run(cmd, capture_output=True, text=True)
                if r.returncode != 0:
                    raise RuntimeError(f"link {name} failed:\n{r.stdout}\n{r.stderr}")
                if verbose:
                    print(f"  linked {out.relative_to(ROOT)}", flush=True)


def ensure_built() -> Path:
    """Build if the library is missing or older than any source (cheap check)."""
    if LIB.exists():
        newest = max(
            (p.stat().st_mtime for p in CSRC.glob("**/*") if p.is_file()),
            default=0,
        )
        if LIB.stat().st_mtime >= newest:
            return LIB
    return build(verbose=False)


if __name__ == "__main__":
    import argparse

    ap = argparse.ArgumentParser()
    ap.add_argument("--force", action="store_true")
    ap.add_argument("--no-bins", action="store_true")
    ap.add_argument("--jobs", type=int, default=None)
    a = ap.parse_args()
    build(force=a.force, bins=not a.no_bins, jobs=a.jobs)
