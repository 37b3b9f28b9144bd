"""Host builds of the device code the CPU tests run: tests/emu/<name>.cu compiled with nvcc for the host only."""
import atexit
import ctypes
import os
import shutil
import subprocess
import tempfile

EMU = os.path.join(os.path.dirname(os.path.abspath(__file__)), "emu")
_libraries = {}


def host_library(name) -> ctypes.CDLL:
    """tests/emu/<name>.cu as a shared library, compiled once per process into a temporary directory."""
    if name not in _libraries:
        tmp = tempfile.mkdtemp(prefix=f"{name}_")
        atexit.register(shutil.rmtree, tmp, ignore_errors=True)
        cmd = ["nvcc", "-O2", "-std=c++17", "-Xcompiler", "-fPIC", "-shared", "-o", os.path.join(tmp, f"lib{name}.so"),
               os.path.join(EMU, f"{name}.cu")]
        proc = subprocess.run(cmd, capture_output=True, text=True)
        if proc.returncode != 0:
            raise RuntimeError("nvcc failed:\n" + " ".join(cmd) + "\n" + proc.stdout + proc.stderr)
        _libraries[name] = ctypes.CDLL(cmd[-2])
    return _libraries[name]
