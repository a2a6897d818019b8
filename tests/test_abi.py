"""CPU: the C-ABI library loads and exports every symbol include/b2v.h declares (no compute calls
without a GPU), and the product never routes through the oracle."""

import ctypes
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _declared_symbols():
    txt = open(os.path.join(ROOT, "include", "b2v.h")).read()
    txt = re.sub(r"/\*.*?\*/", "", txt, flags=re.S)
    return sorted(set(re.findall(r"\b(b2v_[a-z_0-9]+)\s*\(", txt)))


def test_header_symbols_all_exported():
    from pyslam_b200 import _lib
    assert os.path.exists(_lib.LIB_PATH), "libb2v.so was not built"
    L = ctypes.CDLL(_lib.LIB_PATH)
    declared = _declared_symbols()
    assert len(declared) >= 30
    for name in declared:
        assert hasattr(L, name), f"{name} declared in include/b2v.h but not exported"
    assert sorted(_lib.EXPORTED_SYMBOLS) == declared
    assert L.b2v_version() >= 100


def test_library_is_sm90a_and_uses_128bit_cas():
    import shutil
    import subprocess
    from pyslam_b200 import _lib
    cuobjdump = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(cuobjdump):
        pytest.skip("cuobjdump not available")
    out = subprocess.run([cuobjdump, "-lelf", _lib.LIB_PATH], capture_output=True, text=True).stdout
    assert "sm_90a" in out and "sm_100" not in out
    sass = subprocess.run([cuobjdump, "-sass", _lib.LIB_PATH], capture_output=True, text=True).stdout
    assert "allocate_kernel" in sass and "integrate_kernel" in sass
    assert "ATOMG.E.CAS.128" in sass  # 16-byte hash-table entries are inserted with one 128-bit CAS
    assert "UTMALDG.2D" in sass       # depth / colour / lambda tiles are staged by TMA in the allocate kernels
    assert "MATCH.ANY" in sass        # warp-level de-duplication of block inserts (point-average / semantic grids)
    for kernel in ("integrate_group_kernel", "allocate_group_kernel", "mesh_", "sem_runs_kernel", "sem_assoc_kernel",
                   "remap_u8c3_linear_kernel", "shadow_hist_kernel", "depth_u16_to_f32_kernel"):
        assert kernel in sass, kernel


def test_product_does_not_import_oracle():
    """The product path must never route through the CPU oracle (or any CPU fallback)."""
    pkg = os.path.join(ROOT, "pyslam_b200")
    for dirpath, _, files in os.walk(pkg):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".h", ".cpp")):
                src = open(os.path.join(dirpath, f)).read()
                assert not re.search(r"^\s*(from|import)\s+oracle\b", src, flags=re.M), f
                assert "liboracle" not in src and "libref_grid" not in src, f


def test_missing_library_fails_loudly(monkeypatch):
    from pyslam_b200 import _lib
    monkeypatch.setattr(_lib, "_lib", None)
    monkeypatch.setattr(_lib, "LIB_PATH", os.path.join(ROOT, "pyslam_b200", "does_not_exist.so"))
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        _lib.load()


def test_no_gpu_means_an_error_not_a_fallback():
    """Without a CUDA device every product entry point must fail loudly - there is no CPU path to fall back to."""
    from tests._util import has_gpu
    if has_gpu():
        pytest.skip("a GPU is present")
    import numpy as np
    import pyslam_b200 as P
    with pytest.raises(RuntimeError):
        P.B200TsdfVolume(0.01, 0.04, 4.0, capacity_blocks=64)
    with pytest.raises(RuntimeError):
        P.VoxelBlockGrid(0.05, 8, capacity_blocks=64)
    with pytest.raises(RuntimeError):
        P.VoxelBlockSemanticGrid(0.05, 8, capacity_blocks=64)
    with pytest.raises(RuntimeError):
        P.VoxelBlockSemanticProbabilisticGrid(0.05, 8, capacity_blocks=64)
    with pytest.raises(RuntimeError):
        P.filter_shadow_points(np.ones((8, 8), np.float32))
    with pytest.raises(RuntimeError):
        P.remap(np.zeros((4, 4, 3), np.uint8), np.zeros((4, 4), np.float32), np.zeros((4, 4), np.float32))


def test_header_is_plain_c_and_links_against_the_library(tmp_path):
    """include/b2v.h must be consumable from C (the boundary is a C ABI, no C++ or torch types): a C11 translation
    unit that takes the address of every declared entry point compiles with -Wall -Werror -pedantic and links
    against libb2v.so."""
    import shutil
    import subprocess
    from pyslam_b200 import _lib
    gcc = "/usr/bin/gcc" if os.path.exists("/usr/bin/gcc") else shutil.which("gcc")
    if not gcc:
        pytest.skip("gcc not available")
    header = open(os.path.join(ROOT, "include", "b2v.h")).read()
    names = sorted(set(re.findall(r"\b(b2v_[a-z0-9_]+)\s*\(", header)))
    src = tmp_path / "abi_check.c"
    body = "\n".join(f"    table[{i}] = (void (*)(void))&{n};" for i, n in enumerate(names))
    src.write_text('#include "b2v.h"\n#include <stdio.h>\nint main(void) {\n'
                   f"    void (*table[{len(names)}])(void);\n{body}\n"
                   f'    printf("%d %d\\n", b2v_version(), table[{len(names) - 1}] != 0);\n    return 0;\n}}\n')
    exe = tmp_path / "abi_check"
    libdir = os.path.dirname(_lib.LIB_PATH)
    cmd = [gcc, "-std=c11", "-Wall", "-Wextra", "-Werror", "-pedantic",
           "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe), "-L", libdir, "-l:libb2v.so",
           f"-Wl,-rpath,{libdir}"]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    out = subprocess.run([str(exe)], capture_output=True, text=True)
    assert out.returncode == 0 and int(out.stdout.split()[0]) >= 100


def test_voxel_block_grid_duck_type_is_complete():
    """SURVEY.md 8b duck-type B: every method the reference binds on `volumetric.VoxelBlockGrid`
    (cpp/volumetric/volumetric_grid_module.h:732-935, 977-978) exists on the mirror, plus `TBBUtils`
    (volumetric_module.cpp:43-50)."""
    import pyslam_b200 as P
    for name in ("integrate", "get_voxels", "get_points", "get_colors", "clear", "reset", "size", "empty", "num_blocks",
                 "get_block_size", "get_total_voxel_count", "get_voxels_in_bb", "get_voxels_in_camera_frustrum", "carve",
                 "remove_low_count_voxels", "remove_low_confidence_voxels"):
        assert callable(getattr(P.VoxelBlockGrid, name)), name
    for cls in (P.VoxelBlockSemanticGrid, P.VoxelBlockSemanticProbabilisticGrid):
        for name in ("integrate", "integrate_segment", "get_voxels", "get_object_segments", "get_class_segments",
                     "merge_segments", "remove_segment", "remove_low_confidence_segments", "get_ids", "carve",
                     "assign_object_ids_to_instance_ids", "set_depth_threshold", "clear", "reset"):
            assert callable(getattr(cls, name)), (cls.__name__, name)
    P.TBBUtils.set_max_threads(6)
    assert P.TBBUtils.get_max_threads() == 6
