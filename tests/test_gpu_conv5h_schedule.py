"""K-D5h (csrc/pm_conv5.cu, stride-1 halo form) work schedule: 8 x 8 output units walked independently by the two consumer
warpgroups, and the shared-memory plan the launcher picks per layer.

The CPU part checks the plan of every layer the network sends to K-D5h against the H100's 227 KB per-block limit.  The GPU
part runs one shape per plan (resident filter / streamed ring, one or two staging buffers, one or two plane sets), with
fewer units than SMs, many units per CTA, maps that are not a multiple of 8, several images, dilations 1 to 6 and Cout
16 / 18 / 64, against a float64 convolution and against a rerun of itself (bit-identical)."""
import ctypes

import pytest
import torch
import torch.nn.functional as F

from patchmatchnet_b200 import _native, ops

H100_SMEM_OPTIN = 227 * 1024

# dilation of each (Cin, Cout, KS, stride) layer of ops.TC5H_LAYERS in the network (FeatureNet dil 1, the offset convs of stages
# 3 / 2 / 1 dil 2 / 4 / 6)
NET_DILATIONS = {(64, 32, 3, 1): (2,), (64, 18, 3, 1): (2,), (32, 16, 3, 1): (4,), (32, 18, 3, 1): (4,), (16, 18, 3, 1): (6,)}


def plan_of(cin, cout, ks, dil, units, sms=132, optin=H100_SMEM_OPTIN):
    out = (ctypes.c_int * 6)()
    rc = _native.lib().pmb200_conv2d_tc5h_plan(cin, cout, ks, dil, units, sms, optin, out)
    assert rc == 0, _native.lib().pmb200_last_error().decode()
    sbufs, wstages, resident, smem, ctas, psets = list(out)
    return {"sbufs": sbufs, "wstages": wstages, "resident": resident, "smem": smem, "ctas": ctas, "psets": psets}


def units_of(N, H, W):
    return N * ((H + 7) // 8) * ((W + 7) // 8)  # 'same' padding: the output is H x W


@pytest.mark.parametrize("key", sorted(ops.TC5H_LAYERS))
def test_plan_of_every_network_layer_fits_h100(key):
    cin, cout, ks, _ = key
    for dil in NET_DILATIONS.get(key, (1,)):
        for units in (1, 132, 133, 6400):  # one plane set up to one unit per SM of an H100, two beyond
            p = plan_of(cin, cout, ks, dil, units)
            assert p["smem"] <= H100_SMEM_OPTIN, (key, dil, p)
            assert p["psets"] == (1 if units <= 132 else 2)
            assert p["sbufs"] in (1, 2) and 1 <= p["ctas"] <= 4
            assert p["wstages"] == ks * ks if p["resident"] else 2 <= p["wstages"] <= min(8, ks * ks), p
            # as many CTAs per SM as the SM's shared memory holds, each with the 1 KB the driver reserves per block
            assert p["ctas"] * (p["smem"] + 1024) <= H100_SMEM_OPTIN + 1024 and (p["ctas"] == 4 or (p["ctas"] + 1) * (p["smem"] + 1024) > H100_SMEM_OPTIN + 1024)


# (name, N, H, W, Cin, Cout, KS, dil, relu, plan on an H100: (resident filter, staging buffers, plane sets))
CASES = [
    ("resident_two_staging_many_units", 5, 256, 320, 16, 16, 3, 1, True, (1, 2, 2)),
    ("resident_two_staging_dil6", 2, 61, 75, 16, 18, 3, 6, False, (1, 2, 2)),
    ("resident_one_staging_many_units_dil4", 2, 130, 150, 32, 16, 3, 4, False, (1, 1, 2)),
    ("resident_one_plane_set_dil4", 1, 45, 67, 32, 16, 3, 4, False, (1, 1, 1)),
    ("resident_one_plane_set_cout32", 3, 29, 43, 32, 32, 3, 1, True, (1, 1, 1)),
    ("resident_1x1", 3, 19, 27, 64, 16, 1, 1, False, (1, 1, 1)),
    ("ring_one_staging_many_units_cout64", 5, 64, 80, 64, 64, 3, 1, True, (0, 1, 2)),
    ("ring_two_staging_many_units_dil2", 3, 70, 90, 32, 64, 3, 2, True, (0, 2, 2)),
    ("ring_for_two_ctas_cout32", 2, 70, 90, 32, 32, 3, 1, True, (0, 2, 2)),
    ("ring_one_plane_set_cout64", 2, 37, 53, 64, 64, 3, 1, True, (0, 1, 1)),
    ("ring_one_plane_set_fewer_units_than_sms", 1, 37, 45, 64, 18, 3, 2, False, (0, 1, 1)),
    ("ring_one_plane_set_dil2", 1, 64, 80, 64, 32, 3, 2, False, (0, 1, 1)),
]


def test_cases_cover_every_plan():
    seen = set()
    for (name, N, H, W, cin, cout, ks, dil, relu, want) in CASES:
        p = plan_of(cin, cout, ks, dil, units_of(N, H, W))
        assert (p["resident"], p["sbufs"], p["psets"]) == want, name
        seen.add(want)
    assert seen == {(1, 2, 2), (1, 1, 2), (1, 1, 1), (0, 1, 2), (0, 2, 2), (0, 1, 1)}


def _inputs(N, H, W, cin, cout, ks, seed):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(N, cin, H, W, generator=g)
    w = torch.randn(cout, cin, ks, ks, generator=g) / (cin * ks * ks) ** 0.5
    b = torch.randn(cout, generator=g)
    return x, w, b


def _scaled_err(got, want):
    return float((got.double() - want).abs().max() / want.abs().max().clamp_min(1e-6))


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_gpu_conv5h_schedule_matches_float64(case):
    name, N, H, W, cin, cout, ks, dil, relu, want_plan = case
    dev = "cuda:0"
    props = torch.cuda.get_device_properties(0)
    p = plan_of(cin, cout, ks, dil, units_of(N, H, W), props.multi_processor_count, props.shared_memory_per_block_optin)
    assert (p["resident"], p["sbufs"], p["psets"]) == want_plan or props.multi_processor_count != 132, (name, p)
    pad = dil * (ks - 1) // 2
    x, w, b = _inputs(N, H, W, cin, cout, ks, sum(map(ord, name)))
    ref = F.conv2d(x.double(), w.double(), b.double(), 1, pad, dil)
    ref = ref.relu() if relu else ref
    xd = x.to(dev).contiguous(memory_format=torch.channels_last)
    fw = ops.pack_conv_filter_tc5h(w.to(dev))
    got = ops.conv2d_tc5(xd, fw, b.to(dev), cout, ks, 1, pad, dil, relu=relu, halo=True)
    again = ops.conv2d_tc5(xd, fw, b.to(dev), cout, ks, 1, pad, dil, relu=relu, halo=True)
    torch.cuda.synchronize()
    assert got.shape == ref.shape
    err = _scaled_err(got.cpu(), ref)
    assert err <= 1e-5, f"{name}: scaled max err {err:.3e}"
    assert torch.equal(got, again), f"{name}: a rerun differs"


@pytest.mark.gpu
def test_gpu_conv5h_writes_a_channel_slice():
    dev = "cuda:0"
    N, H, W, cin, cout, ks, dil = 2, 27, 35, 64, 18, 3, 2
    x, w, b = _inputs(N, H, W, cin, cout, ks, 5)
    ref = F.conv2d(x.double(), w.double(), b.double(), 1, dil, dil)
    out = torch.full((N, 40, H, W), 7.0, device=dev).contiguous(memory_format=torch.channels_last)
    ops.conv2d_tc5(x.to(dev).contiguous(memory_format=torch.channels_last), ops.pack_conv_filter_tc5h(w.to(dev)), b.to(dev), cout, ks, 1,
                   dil, dil, out=out, out_channel_offset=8, halo=True)
    torch.cuda.synchronize()
    got = out.cpu()
    assert _scaled_err(got[:, 8:8 + cout], ref) <= 1e-5
    assert bool((got[:, :8] == 7.0).all()) and bool((got[:, 8 + cout:] == 7.0).all())
