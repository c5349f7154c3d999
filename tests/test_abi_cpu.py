"""CPU-only: the C-ABI library loads and exports exactly the symbols include/b200t5.h declares;
entry points that need a GPU fail loudly instead of falling back."""
import ctypes as C
import re
import subprocess
from pathlib import Path

import pytest

from anyscale_workshop_nyc_2023_b200 import _lib

ROOT = Path(__file__).resolve().parents[1]


def declared_symbols():
    text = (ROOT / "include" / "b200t5.h").read_text()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(b200t5_[a-z0-9_]+)\s*\(", text)))


@pytest.mark.parametrize("flavour", ["bf16", "fp16"])
def test_every_declared_symbol_is_exported_and_bound(flavour):
    """Both builds of the library (bf16 contract, fp16 contract) export the whole C ABI."""
    lib = _lib.load(flavour)
    names = declared_symbols()
    assert len(names) >= 18
    exported = subprocess.run(["nm", "-D", "--defined-only", str(_lib.LIB_PATHS[flavour])], capture_output=True, text=True).stdout
    for n in names:
        assert re.search(rf"\bT {n}\b", exported), f"{n} not exported"
        assert n in _lib.SIGNATURES, f"{n} declared in the header but not bound in _lib.py"
        getattr(lib, n)
    assert sorted(_lib.SIGNATURES) == names
    assert ("fp16" in lib.b200t5_version().decode()) == (flavour == "fp16")


@pytest.mark.parametrize("flavour", ["bf16", "fp16"])
def test_library_is_sm90a_wgmma(flavour):
    sass = subprocess.run(["cuobjdump", "-sass", str(_lib.LIB_PATHS[flavour])], capture_output=True, text=True).stdout
    assert "sm_90a" in sass
    assert "sm_100" not in sass
    for needle in ("HGMMA", "UTMALDG", "SYNCS"):
        assert needle in sass


def test_no_gpu_means_loud_failure_not_fallback():
    torch = pytest.importorskip("torch")
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    lib = _lib.load()
    cfg = _lib.Config(vocab_size=384, d_model=128, d_kv=64, d_ff=256, num_heads=2, num_layers=2, num_decoder_layers=2,
                      relative_attention_num_buckets=32, relative_attention_max_distance=128, layer_norm_epsilon=1e-6,
                      pad_token_id=0, eos_token_id=1, decoder_start_token_id=0, is_gated_gelu=1, scale_decoder_outputs=0)
    h = C.c_void_p()
    rc = lib.b200t5_create(C.byref(cfg), 0, C.byref(h))
    assert rc == _lib.ENODEV and not h.value
    assert "no CPU fallback" in _lib.last_error()
    from anyscale_workshop_nyc_2023_b200.modeling import B200T5ForConditionalGeneration
    from anyscale_workshop_nyc_2023_b200.workload import checkpoint_dir

    with pytest.raises(RuntimeError, match="no CPU fallback"):
        B200T5ForConditionalGeneration.from_pretrained(checkpoint_dir("tiny", seed=1))


def test_config_validation_is_host_side():
    lib = _lib.load()
    bad = _lib.Config(vocab_size=384, d_model=128, d_kv=32, d_ff=256, num_heads=2, num_layers=2, num_decoder_layers=2,
                      relative_attention_num_buckets=32, relative_attention_max_distance=128, layer_norm_epsilon=1e-6,
                      pad_token_id=0, eos_token_id=1, decoder_start_token_id=0, is_gated_gelu=1, scale_decoder_outputs=0)
    h = C.c_void_p()
    assert lib.b200t5_create(C.byref(bad), 0, C.byref(h)) == _lib.EINVAL
    assert "d_kv" in _lib.last_error()


def test_public_header_is_plain_c(tmp_path):
    """include/b200t5.h is the whole boundary: it must compile as C99 and as C++ with nothing but the standard
    headers (no torch, no CUDA types in the signatures)."""
    src = tmp_path / "hdr.c"
    src.write_text('#include "b200t5.h"\nint main(void) { return sizeof(b200t5_config) == 0; }\n')
    inc = str(ROOT / "include")
    for cmd in (["gcc", "-std=c99", "-Wall", "-Wextra", "-pedantic", "-Werror", "-fsyntax-only", "-I", inc, str(src)],
                ["g++", "-std=c++17", "-Wall", "-Werror", "-fsyntax-only", "-I", inc, "-x", "c++", str(src)]):
        proc = subprocess.run(cmd, capture_output=True, text=True)
        assert proc.returncode == 0, proc.stderr
    code = re.sub(r"/\*.*?\*/", "", (ROOT / "include" / "b200t5.h").read_text(), flags=re.S)  # declarations without comments
    assert "torch" not in code.lower() and "cudaStream_t" not in code and "at::" not in code
    assert re.findall(r"#include\s*[<\"]([^>\"]+)", code) == ["stdint.h"]
