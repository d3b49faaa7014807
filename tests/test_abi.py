"""The C-ABI shared library loads without a GPU and exports every symbol include/*.h declares."""
import ctypes
import re

from conftest import ROOT


def _declared():
    text = (ROOT / "include" / "kdiffusion_b200.h").read_text()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(kdb_[a-z0-9_]+)\s*\(", text)))


def test_header_symbols_exported_and_bound():
    from k_diffusion import _native
    names = _declared()
    assert len(names) >= 25
    handle = ctypes.CDLL(str(_native.LIB_PATH))
    for n in names:
        assert hasattr(handle, n), f"{n} declared in the header but not exported"
    assert set(names) == set(_native.SIGNATURES), set(names) ^ set(_native.SIGNATURES)
    assert _native.lib().kdb_abi_version() == _native.ABI_VERSION


def test_error_reporting_without_gpu():
    from k_diffusion import _native
    L = _native.lib()
    rc = L.kdb_solver_lincomb(None, None, 0, None, 0, None)
    assert rc == -1 and b"n_in" in L.kdb_last_error()
    cfg = _native.KdbModelConfig()
    h = ctypes.c_void_p()
    assert L.kdb_model_create(ctypes.byref(cfg), ctypes.byref(h)) == -1      # n_levels = 0
    assert _native.launch_count() == 0 or _native.launch_count() > 0        # callable


def test_missing_library_fails_loudly(monkeypatch, tmp_path):
    from k_diffusion import _native
    monkeypatch.setattr(_native, "_lib", None)
    monkeypatch.setattr(_native, "LIB_PATH", tmp_path / "nope.so")
    import pytest
    with pytest.raises(_native.NativeLibraryError):
        _native.lib()


def test_every_entry_point_rejects_null_arguments_without_touching_the_gpu():
    """Each compute entry validates its arguments before its first CUDA call: all-NULL / all-zero arguments come back as a
    negative kdb error code with a message (never a crash, never a cudaError from a launch attempt)."""
    from k_diffusion import _native
    L = _native.lib()
    no_args_or_void = {"kdb_abi_version", "kdb_last_error", "kdb_launch_count", "kdb_launch_breakdown", "kdb_model_destroy",
                       "kdb_profile_end", "kdb_profile_gate"}          # gate(0 ns) is a legal request: it launches
    size_queries = {"kdb_model_workspace_bytes": 0, "kdb_model_tap_count": 0}   # return a size, 0 for a NULL model
    checked = 0
    for name, (res, args) in _native.SIGNATURES.items():
        if name in no_args_or_void:
            continue
        zeros = [0.0 if a in (ctypes.c_float, ctypes.c_double) else
                 0 if a in (ctypes.c_int32, ctypes.c_int64, ctypes.c_uint64, ctypes.c_size_t) else None for a in args]
        rc = getattr(L, name)(*zeros)
        if name in size_queries:
            assert rc == size_queries[name], (name, rc)
        else:
            assert rc < 0, f"{name}(NULL...) returned {rc}"
            assert L.kdb_last_error(), name
        checked += 1
    assert checked >= 24


def _engines():
    """(name, native engine, image sizes) of cfg1, the cfg2 model and the four image_v1 U-Net configs; creating an engine needs no GPU"""
    import json
    import k_diffusion as K
    from k_diffusion import _native
    golden = ROOT / "tests" / "golden"
    for stem, sizes in (("cfg1_mnist", [(28, 28)]), ("cfg2_sw256", [(64, 64), (256, 256)])):
        cfg = json.loads((golden / f"{stem}_shapes.json").read_text())["config"]
        yield stem, _native.Engine(K.config.make_model(K.config.load_config(cfg)).engine_spec()), sizes
    for name, meta in sorted(json.loads((golden / "unet_configs.json").read_text()).items()):
        cfg = K.config.load_config(meta["config"])
        model = K.config.make_model(cfg)
        augment = isinstance(model, K.augmentation.KarrasAugmentWrapper)
        spec = (model.inner_model if augment else model).engine_spec(augment)
        yield f"unet {name}", _native.UNetEngine(spec), [tuple(cfg["model"]["input_size"])]


# byte counts of kdb_*_workspace_bytes: a change moves every caller's workspace
WORKSPACE_BYTES = {
    "cfg1_mnist 28x28 B1 prec0": 755712,
    "cfg1_mnist 28x28 B1 prec1": 381952,
    "cfg1_mnist 28x28 B1 vjp": 2415616,
    "cfg1_mnist 28x28 B3 prec0": 2264064,
    "cfg1_mnist 28x28 B3 prec1": 1137664,
    "cfg1_mnist 28x28 B3 vjp": 7239680,
    "cfg2_sw256 64x64 B1 prec0": 2401280,
    "cfg2_sw256 64x64 B1 prec1": 1205248,
    "cfg2_sw256 64x64 B1 vjp": 6569984,
    "cfg2_sw256 64x64 B3 prec0": 7201792,
    "cfg2_sw256 64x64 B3 prec1": 3613696,
    "cfg2_sw256 64x64 B3 vjp": 19705856,
    "cfg2_sw256 256x256 B1 prec0": 38405120,
    "cfg2_sw256 256x256 B1 prec1": 19268608,
    "cfg2_sw256 256x256 B1 vjp": 105089024,
    "cfg2_sw256 256x256 B3 prec0": 115213312,
    "cfg2_sw256 256x256 B3 prec1": 57803776,
    "cfg2_sw256 256x256 B3 vjp": 315262976,
    "unet 32x32_small 32x32 B1": 11927808,
    "unet 32x32_small 32x32 B3": 35782912,
    "unet 32x32_small_butterflies 32x32 B1": 11927808,
    "unet 32x32_small_butterflies 32x32 B3": 35782912,
    "unet cifar10 32x32 B1": 11927808,
    "unet cifar10 32x32 B3": 35782912,
    "unet mnist 28x28 B1": 8981760,
    "unet mnist 28x28 B3": 26944768,
}


def test_workspace_bytes_of_every_engine():
    from k_diffusion import _native
    L = _native.lib()
    got = {}
    for name, eng, sizes in _engines():
        for (H, W) in sizes:
            for B in (1, 3):
                if name.startswith("unet"):
                    got[f"{name} {H}x{W} B{B}"] = int(L.kdb_unet_workspace_bytes(eng._h, _native.PREC_FP32, B, H, W))
                else:
                    for prec in (_native.PREC_FP32, _native.PREC_BF16):
                        got[f"{name} {H}x{W} B{B} prec{prec}"] = int(L.kdb_model_workspace_bytes(eng._h, prec, B, H, W))
                    got[f"{name} {H}x{W} B{B} vjp"] = int(L.kdb_model_vjp_workspace_bytes(eng._h, B, H, W))
    assert got == WORKSPACE_BYTES


def test_set_tensor_rejects_a_null_shape():
    from k_diffusion import _native
    L = _native.lib()
    data = ctypes.c_void_p(256)       # never dereferenced: set_tensor only records the pointer
    for name, eng, _ in _engines():
        set_tensor = L.kdb_unet_set_tensor if name.startswith("unet") else L.kdb_model_set_tensor
        assert set_tensor(eng._h, b"k", data, None, 2) == -1, name
        assert b"set_tensor" in L.kdb_last_error(), name


def test_header_is_plain_c_and_a_c_program_links(tmp_path):
    """The boundary is a C ABI, not a C++ one: the header compiles as pedantic C99 and a C program that calls into the
    library links against libkdb200.so and runs without a GPU (kdb_abi_version, kdb_last_error, an argument-validation failure)."""
    import shutil
    import subprocess
    import pytest
    from k_diffusion import _native
    if shutil.which("gcc") is None:
        pytest.skip("no gcc")
    src = tmp_path / "abi.c"
    src.write_text('#include <stdio.h>\n#include <string.h>\n#include "kdiffusion_b200.h"\n'
                   'int main(void) {\n'
                   '  if (kdb_abi_version() != KDB_ABI_VERSION) return 1;\n'
                   '  if (kdb_solver_lincomb(NULL, NULL, 0, NULL, 0, NULL) >= 0) return 2;\n'
                   '  if (strlen(kdb_last_error()) == 0) return 3;\n'
                   '  printf("abi %d\\n", kdb_abi_version());\n'
                   '  return 0;\n}\n')
    inc, libdir = str(ROOT / "include"), str(_native.LIB_PATH.parent)
    subprocess.run(["gcc", "-std=c99", "-Wall", "-Wextra", "-pedantic", "-Werror", "-I", inc, "-fsyntax-only", str(src)], check=True)
    exe = tmp_path / "abi"
    subprocess.run(["gcc", "-std=c99", "-I", inc, str(src), "-o", str(exe), "-L", libdir, "-l:" + _native.LIB_PATH.name,
                    "-Wl,-rpath," + libdir, "-Wl,--unresolved-symbols=ignore-in-shared-libs"], check=True)
    out = subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout
    assert out.strip() == f"abi {_native.ABI_VERSION}"


def test_integration_guide_names_every_entry_point():
    """INTEGRATION.md is the reference-side binding guide: it must mention every function the header declares."""
    doc = (ROOT / "INTEGRATION.md").read_text()
    missing = [n for n in _declared() if n not in doc]
    assert not missing, missing
