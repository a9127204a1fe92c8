"""CPU-side checks of the C ABI: the library loads without a GPU / libcuda, exports every symbol
that include/osvos_b200.h declares, and the ctypes table mirrors the header."""
import ctypes
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def lib_path():
    from osvos_pytorch_b200 import build
    return build.build()


def header_functions():
    src = open(os.path.join(ROOT, "include", "osvos_b200.h")).read()
    return sorted(set(re.findall(r"OSVOS_API\s+[\w\s\*]+?\b(osvos_\w+)\s*\(", src)))


def test_header_declares_expected_entry_points():
    names = header_functions()
    for required in ("osvos_version", "osvos_last_error", "osvos_conv3x3", "osvos_conv_first_fwd",
                     "osvos_maxpool2x2_fwd", "osvos_tail_fwd", "osvos_cbce_fwd", "osvos_cbce_bwd",
                     "osvos_pack_conv3x3_weights"):
        assert required in names


def test_library_exports_every_declared_symbol(lib_path):
    lib = ctypes.CDLL(lib_path)
    for name in header_functions():
        assert hasattr(lib, name), f"{name} declared in include/osvos_b200.h but not exported"
    lib.osvos_version.restype = ctypes.c_int
    assert lib.osvos_version() == 100


def test_ctypes_table_matches_header(lib_path):
    from osvos_pytorch_b200 import _native as nat
    assert sorted(nat.SIGNATURES) == header_functions()
    lib = nat.load()
    assert lib.osvos_version() == 100
    # argument validation happens before any CUDA call: NULL args -> OSVOS_ERR_INVALID_ARGUMENT, with a message
    assert lib.osvos_conv3x3(None, None) == 1
    assert b"invalid argument" in lib.osvos_last_error()


@pytest.mark.parametrize("field,rejected_by", [("none", "a->bias"), ("y_hi", "a->cout != 16"), ("y_lo", "a->cout != 16"),
                                               ("relu_mask", "a->cout != 16"), ("colsum", "a->colsum == nullptr")])
def test_conv3x3_16_channel_outputs_are_fp32_features_or_projections(lib_path, field, rejected_by):
    """cout == 16 (side_prep) writes fp32 features and / or projections only; act outputs, ReLU masks and column sums are
    refused.  Validation runs before any CUDA call.  The bias pointer is misaligned in every case, so a call that passes
    the cout == 16 checks (the control, "none") stops at the alignment check and never reaches a kernel."""
    from osvos_pytorch_b200 import _native as nat
    lib = nat.load()
    addr = 1 << 20                                   # placeholder device address, never dereferenced
    a = nat.Conv3x3Args()
    a.x_hi = a.x_lo = a.w_packed = a.y_f32 = addr
    a.bias = addr + 4
    a.n, a.h, a.w, a.cin, a.cout = 1, 8, 8, 64, 16
    if field == "relu_mask":
        a.mask_hi, a.flags = addr, nat.FLAG_RELU_MASK
    elif field != "none":
        setattr(a, field, addr)
    assert lib.osvos_conv3x3(ctypes.byref(a), None) == 1
    msg = lib.osvos_last_error()
    assert b"invalid argument" in msg and rejected_by.encode() in msg, msg


def test_library_reads_only_the_pdl_and_ablation_switches():
    calls, names = 0, set()
    for dirpath, _, files in os.walk(os.path.join(ROOT, "osvos_pytorch_b200", "csrc")):
        for f in files:
            txt = open(os.path.join(dirpath, f)).read()
            calls += len(re.findall(r"\bgetenv\s*\(", txt))
            names |= set(re.findall(r"\bgetenv\s*\(\s*\"(\w+)\"\s*\)", txt))
    assert names == {"OSVOS_PDL", "OSVOS_ABLATE"}
    assert calls == 2                                # every getenv call names its variable literally


def test_product_package_never_imports_the_oracle():
    pkg = os.path.join(ROOT, "osvos_pytorch_b200")
    for dirpath, _, files in os.walk(pkg):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh")):
                txt = open(os.path.join(dirpath, f)).read()
                assert not re.search(r"^\s*(from|import)\s+oracle\b", txt, flags=re.M), f
                assert "/root/reference" not in txt, f


def test_cpu_input_fails_loudly(lib_path):
    import torch
    from osvos_pytorch_b200.networks.vgg_osvos import OSVOS
    net = OSVOS(pretrained=0, verbose=False)
    assert len(net.state_dict()) == 52
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        net(torch.zeros(1, 3, 16, 16))
