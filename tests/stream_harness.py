"""What the GPU stream tests share: the device fixture, the pwgb_debug_get reader, synthetic mel frames, the golden and
synthetic model loaders, and the history-conv kernel cases."""
import ctypes as C
import json

import pytest
import torch

from helpers import golden_weights, load_golden
from oracle import synth


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "gpu tests need a CUDA device"
    import __graft_entry__

    __graft_entry__.build()
    return torch.device("cuda:0")


def debug_get(key, n):
    """the first n ints of libpwgb's debug record ``key`` (pwgb_debug_get): what the last launch of a kind chose"""
    from parallelwavegan_b200 import capi

    v = (C.c_int * n)()
    assert capi.lib().pwgb_debug_get(key, C.cast(v, C.c_void_p), C.sizeof(v)) == 0
    return list(v)


def mels(B, T, seed):
    """(B, T, 80) synthetic mel frames"""
    return synth.randn((B, T, 80), seed)


def golden_model(dev, cls, name, weight_norm=True):
    """(meta, golden arrays, models.<cls> with the weights of tests/golden/<name>.npz, in eval mode on dev)"""
    from parallelwavegan_b200 import models

    meta, g = load_golden(name)
    m = getattr(models, cls)(**json.loads(json.dumps(meta["kwargs"])))
    m.load_state_dict(golden_weights(meta), strict=True)
    if not weight_norm:
        m.remove_weight_norm()
    return meta, g, m.to(dev).eval()


def synthetic_model(dev, cls, kwargs, seed, gain, weight_norm=True):
    """models.<cls>(**kwargs) with synthetic weights (oracle.synth), in eval mode on dev"""
    from parallelwavegan_b200 import models

    m = getattr(models, cls)(**json.loads(json.dumps(kwargs)))
    m.load_state_dict(synth.synth_state_dict([(k, tuple(v.shape)) for k, v in m.state_dict().items()], seed, gain))
    if not weight_norm:
        m.remove_weight_norm()
    return m.to(dev).eval()


# the history conv's kernel cases
# name: B, cin, cout, K, dilation, n, H, pad_left, replicate flags, epilogue, engine, expected plan
#   plan (tensor cores, pwgb_debug_get(1)): "cp" cp.async-staged, "direct" register path, "win" win_mode, "nco" column chunks
KCASES = {
    "tc_cp_h_eq_pad": (2, 64, 64, 3, 2, 300, 4, 4, None, "plain", "tc", "cp"),
    "tc_cp_h_lt_pad_rep": (3, 32, 48, 7, 1, 200, 3, 6, [1, 0, 1], "res", "tc", "cp"),
    "tc_direct_n_lt_h": (2, 32, 32, 3, 176, 100, 352, 352, [0, 1], "acc", "tc", "direct"),
    "tc_win": (1, 32, 32, 3, 1100, 500, 2200, 2200, None, "plain", "tc", "win"),
    "tc_nco_staged": (3, 32, 256, 11, 5, 700, 50, 50, [1, 0, 0], "res", "tc", "nco"),
    "ffma_h_eq_pad": (2, 16, 8, 3, 3, 257, 6, 6, [0, 1], "plain", "simt", None),
    "ffma_h_lt_pad": (3, 8, 2, 7, 1, 90, 4, 6, [1, 0, 1], "res", "simt", None),
    "ffma_n_lt_h": (2, 4, 16, 11, 5, 20, 50, 50, None, "acc", "simt", None),
    "ffma_tanh": (3, 32, 1, 7, 1, 3000, 6, 6, [0, 1, 1], "tanh", "simt", None),
}
