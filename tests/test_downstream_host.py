"""CPU checks of the concat-conditioned UNetModel and the downstream tasks' Python surface: the oracle against fixtures of the
reference's own modules (scripts/make_cond_goldens.py), the C ABI's refusals (all before a device is needed) and the wrapper
chain the solvers read the condition from."""
import ctypes as C
import types

import pytest
import torch

import lfm_b200
from lfm_b200 import solvers
from oracle import solvers as osol
from oracle import unet as ounet
from tests._util import T, load_golden, rel_l2


@pytest.fixture(scope="module")
def lib():
    from lfm_b200 import _lib, build
    build.build()
    return _lib.load()


def cfg_from_golden(g):
    return ounet.UNetConfig(image_size=int(g["cfg_image_size"]), in_channels=int(g["cfg_in_channels"]),
                            model_channels=int(g["cfg_model_channels"]), out_channels=int(g["cfg_out_channels"]),
                            num_res_blocks=int(g["cfg_num_res_blocks"]),
                            attention_resolutions=tuple(int(v) for v in g["cfg_attention_resolutions"]),
                            channel_mult=tuple(int(v) for v in g["cfg_channel_mult"]), num_heads=int(g["cfg_num_heads"]),
                            num_head_channels=int(g["cfg_num_head_channels"]))


@pytest.mark.parametrize("name,in_ch", [("unet_inpaint_mini", 9), ("unet_semantic_mini", 8)])
def test_oracle_matches_conditioned_reference_fixture(name, in_ch):
    g = load_golden(name)
    cfg = cfg_from_golden(g)
    assert cfg.in_channels == in_ch and g["cond"].shape[1] == in_ch - 4
    sd = ounet.synthetic_state_dict(cfg, int(g["weight_seed"]))
    assert tuple(sd["input_blocks.0.0.weight"].shape) == (cfg.model_channels, in_ch, 3, 3)
    cond = T(g["cond"])
    f = lambda t, x: ounet.unet_forward(sd, cfg, t, torch.cat([x, cond], 1))  # noqa: E731
    v = f(T(g["t_vec"]), T(g["z"]))
    assert rel_l2(v, g["v"]) < 2e-5 and float(abs(g["v"]).mean()) > 1e-2
    assert rel_l2(osol.tdq_euler(f, T(g["z"]), float(g["euler_step"]))[0], g["euler"]) < 2e-5


def test_spatial_rescaler_matches_reference_fixture():
    g = load_golden("spatial_rescaler")
    m = lfm_b200.SpatialRescaler(n_stages=3, in_channels=19, out_channels=4, multiplier=0.5)
    assert list(m.state_dict()) == ["channel_mapper.weight"]
    m.load_state_dict({"channel_mapper.weight": T(g["weight"])}, strict=True)
    seg = T(g["seg"]).long()
    with torch.no_grad():
        out = m(torch.nn.functional.one_hot(seg, 19).permute(0, 3, 1, 2).float())
    assert out.shape == (2, 4, 32, 32)
    assert rel_l2(out, g["out"]) < 1e-6


def test_unet_model_takes_concatenated_channels():
    net = lfm_b200.UNetModel(image_size=16, in_channels=9, model_channels=128, out_channels=4, num_res_blocks=1,
                             attention_resolutions=(2,), channel_mult=(1, 2), num_heads=2, use_scale_shift_norm=True)
    sd = net.state_dict()
    assert tuple(sd["input_blocks.0.0.weight"].shape) == (128, 9, 3, 3) and tuple(sd["out.2.weight"].shape) == (4, 128, 3, 3)
    with pytest.raises(RuntimeError):
        net(0.5, torch.zeros(1, 9, 16, 16))                          # no CPU path


class _Net(lfm_b200.network._NativeNet):
    """Stands in for a network: the wrapper walk only needs the type and the channel counts."""

    def __init__(self, in_channels=9):
        super().__init__()
        self.in_channels, self.out_channels = in_channels, 4


class _NFECount(torch.nn.Module):
    def __init__(self, model):
        super().__init__()
        self.model = model


def test_wrapper_chain_hands_its_condition_to_the_solver():
    net = _Net()
    c1, c2 = torch.randn(2, 3, 8, 8), torch.randn(2, 2, 8, 8)
    w = lfm_b200.WrapperCondFlow(net, torch.cat([c1, c2], 1))
    assert solvers._unwrap(w) is net and torch.equal(solvers._condition(w), torch.cat([c1, c2], 1))
    # nested: WrapperCondFlow(WrapperCondFlow(net, c2), c1)(t, x) = net(t, cat([x, c1, c2], 1))
    nested = _NFECount(lfm_b200.WrapperCondFlow(lfm_b200.WrapperCondFlow(net, c2), c1))
    nested.count_nfe = True
    assert solvers._unwrap(nested) is net and torch.equal(solvers._condition(nested), torch.cat([c1, c2], 1))
    # the concatenation the wrappers compute, with a torch stand-in for the network
    seen = {}

    class Probe(torch.nn.Module):
        def forward(self, t, x):
            seen["x"] = x
            return x[:, :4]

    x = torch.randn(2, 4, 8, 8)
    lfm_b200.WrapperCondFlow(lfm_b200.WrapperCondFlow(Probe(), c2), c1)(0.5, x)
    assert torch.equal(seen["x"], torch.cat([x, c1, c2], 1))
    assert solvers._condition(_NFECount(net)) is None
    with pytest.raises(ValueError):
        solvers._set_condition(net, None, None, x)                 # a 9-channel network without a condition
    with pytest.raises(ValueError):
        solvers._set_condition(net, None, c1, x)                   # 3 channels where the network takes 5


def test_downstream_sample_from_model_signature():
    net = _Net()
    w = lfm_b200.WrapperCondFlow(net, torch.zeros(1, 5, 8, 8))
    args = types.SimpleNamespace(method="dopri8", atol=1e-5, rtol=1e-5, compute_fid=False)
    with pytest.raises(NotImplementedError):
        lfm_b200.downstream.sample_from_model(w, torch.zeros(1, 4, 8, 8), args)
    assert w.count_nfe is True                                       # set as the reference does; harmless here


def unet_desc(lib_mod, in_ch=4, out_ch=4):
    return lib_mod.UnetDesc(16, in_ch, 128, out_ch, 1, 1, (C.c_int32 * 8)(2), 2, (C.c_int32 * 8)(1, 2), 2, -1, 0)


def test_conditioned_create_refusals(lib):
    from lfm_b200 import _lib
    ctx = C.c_void_p()
    for in_ch, out_ch in ((3, 4), (17, 4), (9, 5)):
        assert lib.lfm_create_unet(C.byref(unet_desc(_lib, in_ch, out_ch)), 0, C.byref(ctx)) != 0
        assert "in_channels must be in [4, 16] and out_channels 4" in _lib.last_error(), _lib.last_error()
    edm = _lib.EdmDesc(16, 9, 4, 0, 128, 2, (C.c_int32 * 8)(1, 2), 1, 1, (C.c_int32 * 8)(8))
    assert lib.lfm_create_edm(C.byref(edm), 0, C.byref(ctx)) != 0 and "in/out channels must be 4" in _lib.last_error()
    dit = _lib.ModelDesc(0, 32, 2, 9, 256, 2, 4, 1024, 1)
    assert lib.lfm_create(C.byref(dit), 0, C.byref(ctx)) != 0 and "in_channels must be 4" in _lib.last_error()


def test_conditioned_entries_refuse_bad_arguments(lib):
    from lfm_b200 import _lib

    def refused(rc, word):
        assert rc != 0
        assert word in _lib.last_error(), _lib.last_error()

    refused(lib.lfm_set_condition(None, None, 1, 5, None), "null ctx")
    # lfm_dbg_conv_in(a, a_ch, a_stride, b, b_ch, b_stride, w, bias, out, B, side, Cout, stream)
    ci = lib.lfm_dbg_conv_in
    d = C.c_void_p(64)   # never dereferenced: each call is refused on its arguments
    refused(ci(d, 2, 2 * 256, None, 0, 0, d, d, d, 1, 16, 128, None), "a_ch + b_ch")
    refused(ci(d, 9, 9 * 256, d, 8, 8 * 256, d, d, d, 1, 16, 128, None), "a_ch + b_ch")
    refused(ci(d, 0, 0, d, 4, 4 * 256, d, d, d, 1, 16, 128, None), "a_ch")
    refused(ci(d, 4, 4 * 512 * 512, None, 0, 0, d, d, d, 1, 512, 128, None), "side")
    refused(ci(d, 16, 16 * 65536, None, 0, 0, d, d, d, 1, 256, 128, None), "side")
    refused(ci(d, 4, 100, None, 0, 0, d, d, d, 1, 16, 128, None), "a_stride")
    refused(ci(d, 4, 1024, d, 5, 100, d, d, d, 1, 16, 128, None), "b_stride")
    refused(ci(d, 4, 1024, None, 0, 0, d, d, d, 1, 16, 0, None), "Cout")
    refused(ci(d, 4, 1024, None, 0, 0, d, d, d, 0, 16, 128, None), "B")
    refused(ci(d, 4, 1024, None, 5, 1280, d, d, d, 1, 16, 128, None), "NULL")
    refused(ci(d, 4, 1024, None, 0, 0, d, None, d, 1, 16, 128, None), "NULL")
