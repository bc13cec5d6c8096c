"""The GQA group bound of the two decode entry points (b200_attn_decode, b200_attn_decode_fused): the wgmma decode
kernel takes groups of 1 to 16 query heads per kv head.  A larger group is refused by the argument checks, before
any CUDA call; groups of 9 to 16 pass every check, so without a device only the missing device stops them.
Fake device addresses, as in test_attn_entry_cpu.py, so the file only runs where there is no device."""
import pytest
import torch

from test_attn_entry_cpu import ALL_WORDS, BS, D, _call, _decode_args

pytestmark = pytest.mark.skipif(torch.cuda.is_available(), reason="fake device pointers: CPU-only test")

GROUP_WORDS = "GQA group size"


def _group_args(native_lib, phase, hq, hkv):
    a = _decode_args(native_lib, phase == "fused")
    a.update(hq=hq, hkv=hkv, q_rs=(hq + 2 * hkv) * D, k_rs=(hq + 2 * hkv) * D, v_rs=(hq + 2 * hkv) * D,
             ws_bytes=native_lib.b200_attn_workspace_bytes(BS, hq, D))
    return a


@pytest.mark.parametrize("phase", ["decode", "fused"])
@pytest.mark.parametrize("hq,hkv", [(17, 1), (32, 1), (34, 2), (256, 8)])
def test_group_above_16_is_refused(b200, native_lib, phase, hq, hkv):
    launches = native_lib.b200_launch_count()
    assert _call(native_lib, phase, _group_args(native_lib, phase, hq, hkv)) != 0
    err = native_lib.b200_last_error().decode()
    assert GROUP_WORDS in err and "wgmma" in err and "16" in err, err
    assert native_lib.b200_launch_count() == launches


@pytest.mark.parametrize("phase", ["decode", "fused"])
@pytest.mark.parametrize("hq,hkv", [(9, 1), (12, 1), (16, 1), (24, 2), (96, 8), (128, 8)])
def test_group_of_9_to_16_passes_every_check(b200, native_lib, phase, hq, hkv):
    launches = native_lib.b200_launch_count()
    assert _call(native_lib, phase, _group_args(native_lib, phase, hq, hkv)) != 0
    err = native_lib.b200_last_error().decode()
    assert GROUP_WORDS not in err and not any(w in err for w in ALL_WORDS), err
    assert native_lib.b200_launch_count() == launches
