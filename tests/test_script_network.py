"""TorchScript deployment of the whole network (reference train.py:50-55 writes `torch.jit.script(model)` as module_%06d.pt,
eval.py:38-39 runs it with torch.jit.load under nn.DataParallel).  CPU tests: the new operators' schemas, compile + save + load
of PatchmatchNet in both precisions, the frozen per-layer decisions, the training-mode error and train.export_module's
archive (no kernel runs).  GPU tests: scripted == eager bit for bit on every request shape the network takes, the scripted stage
in the fp32-accurate mode, each new operator against its ctypes wrapper, the archive in a fresh interpreter, under
nn.DataParallel and from C++, and a trained module_%06d.pt against its checkpoint."""
import io
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from patchmatchnet_b200 import PatchMatch, _native, ops, train
from patchmatchnet_b200.net import PatchmatchNet, load_reference_state
from tests import multisize_cases, pm_cases, scene_cases
from tests.geo_cases import plane_depth

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DEV = "cuda:0"
NET_DEPTH_TOL = 2e-4  # test_network_matches_reference_golden / tests/test_gpu_multisize.py
NEW_OPS = ["conv2d_nhwc_out", "conv2d_tc5", "conv2d_tc5_out", "conv_stem", "refine_low", "refine_full", "upsample2x_add",
           "pack_nhwc_views", "warp_corr_views", "warp_corr_view_weights_views", "warp_corr_score_views_", "device_copy"]


@pytest.fixture(scope="module", autouse=True)
def _ops_loaded():
    _native.build_torch_library()
    _native.load_torch_ops()


@pytest.fixture(params=[False, True], ids=["fp32", "tf32"])
def tf32(request):
    """The precision switch the decisions are frozen under (set before eval()), restored afterwards."""
    old = (torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32)
    torch.backends.cudnn.allow_tf32 = request.param
    torch.backends.cuda.matmul.allow_tf32 = request.param
    yield request.param
    torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = old


def _net(weights, device=None):
    net = PatchmatchNet(**pm_cases.NET_KWARGS)
    load_reference_state(net, weights)
    if device is not None:
        net = net.to(device)
    return net.eval()


def _node_kinds(block):
    kinds = set()
    for n in block.nodes():
        kinds.add(n.kind())
        for b in n.blocks():
            kinds |= _node_kinds(b)
    return kinds


def _round_trip(sm):
    buf = io.BytesIO()
    torch.jit.save(sm, buf)
    buf.seek(0)
    return torch.jit.load(buf, map_location="cpu")


# ---- CPU ---------------------------------------------------------------------------------------------------------------------
def test_new_operators_are_registered_with_schemas():
    for name in NEW_OPS:
        schema = str(getattr(torch.ops.pmb200, name).default._schema)
        assert schema.startswith(f"pmb200::{name}("), schema
    for name in ("conv2d_nhwc_out", "conv2d_tc5_out"):
        assert "Tensor(a!) out" in str(getattr(torch.ops.pmb200, name).default._schema)
    assert "Tensor(a!) xs" in str(torch.ops.pmb200.warp_corr_score_views_.default._schema)
    assert "-> (Tensor, Tensor)" in str(torch.ops.pmb200.pack_nhwc_views.default._schema)
    with pytest.raises((NotImplementedError, RuntimeError)):  # CUDA is the only backend
        torch.ops.pmb200.pack_nhwc_views([torch.zeros(1, 8, 4, 4)])


def test_network_scripts_with_native_calls_only_and_keeps_the_reference_keys(golden_weights, tf32):
    net = _net(golden_weights)
    sm = torch.jit.script(net)
    kinds = _node_kinds(sm.inlined_graph)
    foreign = {k for k in kinds if not k.startswith(("aten::", "pmb200::", "prim::"))}
    assert not foreign, foreign
    assert "prim::PythonOp" not in kinds
    for op in ("pmb200::conv2d_nhwc_out", "pmb200::pack_nhwc_views", "pmb200::warp_corr_score_views_", "pmb200::refine_low",
               "pmb200::conv_stem", "pmb200::upsample2x_add", "pmb200::photometric_confidence"):
        assert op in kinds, op
    back = _round_trip(sm)
    assert sorted(back.state_dict()) == sorted(net.state_dict())  # exactly the reference's keys
    for k, v in back.state_dict().items():
        assert torch.equal(v, net.state_dict()[k]), k


def test_frozen_decisions_are_the_conv_forms_eager_picks(golden_weights, tf32):
    net = _net(golden_weights)
    pairs = [(net.feature, f"conv{i}") for i in range(11)] + [(net.upsample_net, f"conv{i}") for i in range(4)]
    for owner, name in pairs:
        layer = getattr(owner, name)
        c = layer.conv
        prefers = ops.conv_prefers_native(c.in_channels, c.out_channels, c.kernel_size[0])
        assert layer._s_mode == (2 if prefers else 1), name
        assert layer._s_form == ops.conv_form(c.in_channels, c.out_channels, c.kernel_size[0], c.stride[0]), name
        assert layer._s_precision == ops.conv_precision()
    for name in ("output1", "inner1", "inner2", "output2", "output3"):
        c = getattr(net.feature, name)
        assert net.feature._s_plain_form[name] == ops.conv_form(c.in_channels, c.out_channels, 1, 1), name
    assert net.feature._s_stem_fused == (not tf32) and net.upsample_net._s_fused == (not tf32)
    assert net.feature._s_top_down == 2
    for stage in (net.patchmatch_1, net.patchmatch_2, net.patchmatch_3):
        for conv, native, form in ((stage.propa_conv, stage._native_propa, stage._off_propa_form),
                                   (stage.eval_conv, stage._native_eval, stage._off_eval_form)):
            assert native == ops.conv_prefers_native(conv.in_channels, conv.out_channels, 3)
            if native:
                assert form == ops.conv_form(conv.in_channels, conv.out_channels, 3, 1)
    if not tf32:  # the stage offset convs of ops.TC5H_LAYERS take the halo-tile form, as in eager
        assert net.patchmatch_3._off_eval_form == 2 and net.patchmatch_2._off_eval_form == 2
    assert not any(k.startswith("_s_") or "._s_" in k for k in net.state_dict())


def test_scripted_network_is_inference_only(golden_weights):
    sm = torch.jit.script(_net(golden_weights))
    sm.train()
    inp = pm_cases.make_net_inputs(pm_cases.NET_CASE)
    with pytest.raises(Exception, match="inference-only"):
        sm(inp["images"], inp["intrinsics"], inp["extrinsics"], inp["depth_min"], inp["depth_max"])


def test_export_module_writes_a_runnable_network(golden_weights, tmp_path):
    net = PatchmatchNet(**pm_cases.NET_KWARGS)
    load_reference_state(net, golden_weights)
    net.train()
    path = str(tmp_path / "module_000000.pt")
    train.export_module(net, path)
    assert net.training  # the caller's mode is restored
    back = torch.jit.load(path, map_location="cpu")
    assert isinstance(back, torch.jit.ScriptModule) and hasattr(back, "forward")
    assert "pmb200::" in str(back.inlined_graph)
    assert sorted(back.state_dict()) == sorted(net.state_dict())


# ---- GPU ---------------------------------------------------------------------------------------------------------------------
def _requests():
    """name -> (inputs, fixed stage-3 draw): the golden request, B = 2, a size that is not a multiple of 8, mixed sizes."""
    out = {"net_case": pm_cases.make_net_inputs(pm_cases.NET_CASE),
           "batch2": pm_cases.make_net_inputs(dict(B=2, n_views=3, H=64, W=96, seed=41)),
           "not_multiple_of_8": pm_cases.make_net_inputs(dict(B=1, n_views=3, H=61, W=83, seed=42)),
           "mixed_sizes": multisize_cases.make_net_inputs()}
    inp = out["not_multiple_of_8"]
    inp["rand48"] = torch.rand(1, 48, 8, 10, generator=torch.Generator().manual_seed(3))  # after rounding to 64x80
    return out


def _args(inp):
    return ([i.to(DEV) for i in inp["images"]], inp["intrinsics"].to(DEV), inp["extrinsics"].to(DEV), inp["depth_min"].to(DEV),
            inp["depth_max"].to(DEV))


def _run(model, inp):
    with torch.no_grad():
        return model(*_args(inp))


def _assert_same(a, b):
    d0, c0, s0 = a
    d1, c1, s1 = b
    assert torch.equal(d0, d1) and torch.equal(c0, c1)
    assert sorted(s0) == sorted(s1)
    for k in s0:
        assert len(s0[k]) == len(s1[k])
        for x, y in zip(s0[k], s1[k]):
            assert torch.equal(x, y), k


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["net_case", "batch2", "not_multiple_of_8", "mixed_sizes"])
def test_scripted_network_equals_eager(golden_weights, golden_net_case, tf32, name):
    inp = _requests()[name]
    net = _net(golden_weights, DEV)
    rand = inp["rand48"].to(DEV)
    net.patchmatch_3.rand_source = lambda size, device: rand
    sm = torch.jit.script(net)
    sm.patchmatch_3.rand_draw = rand
    eager, scripted = _run(net, inp), _run(sm, inp)
    _assert_same(eager, scripted)
    # seeded draws instead of the fixed one: the same torch.rand stream in both
    net.patchmatch_3.rand_source = None
    sm.patchmatch_3.rand_draw = torch.empty(0)
    torch.cuda.manual_seed(17)
    eager = _run(net, inp)
    torch.cuda.manual_seed(17)
    _assert_same(eager, _run(sm, inp))
    if tf32 or name not in ("net_case", "mixed_sizes"):
        return
    gold = golden_net_case if name == "net_case" else torch.load(os.path.join(REPO, "tests", "golden", "multisize_case.pt"))["net"]
    depth, conf, per_stage = scripted
    assert pm_cases.rel_l1(depth, gold["depth"]) <= NET_DEPTH_TOL
    for s, ds in gold["per_stage"].items():
        for x, y in zip(per_stage[s], ds):
            assert pm_cases.rel_l1(x, y) <= NET_DEPTH_TOL
    assert float((conf.cpu() - gold["confidence"]).abs().max()) <= 5e-2
    assert float((conf.cpu() - gold["confidence"]).abs().mean()) <= 1e-3


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(pm_cases.STAGE_CASES))
def test_scripted_stage_equals_eager_in_the_fp32_accurate_mode(golden_weights, name):
    old = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = False
    try:
        spec = pm_cases.STAGE_CASES[name]
        case = pm_cases.make_stage_inputs(spec)
        mod = PatchMatch(**pm_cases.stage_ctor_kwargs(spec["stage"]))
        mod.load_state_dict(pm_cases.stage_state(golden_weights, spec["stage"]), strict=True)
        mod.eval()
        sm = torch.jit.script(mod)
        mod.to(DEV)
        sm.to(DEV)
        args = [case["ref_feature"].to(DEV), [s.to(DEV) for s in case["src_features"]], case["ref_proj"].to(DEV),
                [m.to(DEV) for m in case["src_projs"]], case["depth_min"].to(DEV), case["depth_max"].to(DEV), case["depth"].to(DEV),
                case["view_weights"].to(DEV)]
        with torch.no_grad():
            torch.cuda.manual_seed(11)
            d0, p0, v0 = mod(*args)
            torch.cuda.manual_seed(11)
            d1, p1, v1 = sm(*args)
    finally:
        torch.backends.cudnn.allow_tf32 = old
    for a, b in zip(d0, d1):
        assert torch.equal(a, b)
    assert torch.equal(p0, p1) and torch.equal(v0, v1)


def _cl(t):
    return t.to(DEV).contiguous(memory_format=torch.channels_last)


@pytest.mark.gpu
def test_new_ops_equal_the_ctypes_wrappers_in_every_conv_form():
    g = torch.Generator().manual_seed(5)
    P = torch.ops.pmb200
    x = _cl(torch.randn(2, 32, 24, 40, generator=g))
    for cout, ks, stride, pad, dil in ((16, 3, 1, 2, 2), (64, 5, 2, 2, 1), (18, 3, 1, 1, 1)):
        w = torch.randn(cout, 32, ks, ks, generator=g) * 0.1
        b = torch.randn(cout, generator=g)
        for prec in (1, 3):
            frag = ops.pack_conv_filter(w, prec)
            want = ops.conv2d_nhwc(x, frag.to(DEV), b.to(DEV), cout, ks, stride, pad, dil, relu=True, precision=prec)
            out = torch.empty_like(want)
            P.conv2d_nhwc_out(x, frag, b, cout, ks, stride, pad, dil, True, prec, False, None, out, 0)  # host filter and bias
            assert torch.equal(out, want)
        for form in (1, 2):
            if form == 2 and stride != 1:
                continue
            filt = ops.pack_conv_filter_for(w, form, 3)
            want = ops.conv2d_tc5(x, filt.to(DEV), b.to(DEV), cout, ks, stride, pad, dil, relu=True, halo=form == 2)
            assert torch.equal(P.conv2d_tc5(x, filt, b, cout, ks, stride, pad, dil, True, form == 2), want)
            wide = torch.zeros(want.shape[0], cout + 8, *want.shape[2:], device=DEV).contiguous(memory_format=torch.channels_last)
            P.conv2d_tc5_out(x, filt, b.to(DEV), cout, ks, stride, pad, dil, True, form == 2, wide, 8)
            assert torch.equal(wide[:, 8:], want) and not wide[:, :8].any()
    # add_up2x, transposed2x and a channel window of a wider output
    fine = _cl(torch.randn(2, 16, 24, 40, generator=g))
    coarse = _cl(torch.randn(2, 32, 12, 20, generator=g))
    frag = ops.pack_conv_filter(torch.randn(32, 16, 1, 1, generator=g), 3).to(DEV)
    want = ops.conv2d_nhwc(fine, frag, None, 32, 1, precision=3, add_up2x=coarse)
    out = torch.empty_like(want)
    P.conv2d_nhwc_out(fine, frag, None, 32, 1, 1, 0, 1, False, 3, False, coarse, out, 0)
    assert torch.equal(out, want)
    low = _cl(torch.randn(2, 8, 12, 20, generator=g))
    frag = ops.pack_conv_filter(torch.randn(8, 8, 3, 3, generator=g), 3, transposed=True).to(DEV)
    a = torch.zeros(2, 16, 24, 40, device=DEV).contiguous(memory_format=torch.channels_last)
    b2 = torch.zeros_like(a)
    ops.conv2d_nhwc(low, frag, None, 8, 3, 1, 1, 1, relu=True, transposed2x=True, out=a, out_channel_offset=8, precision=3)
    P.conv2d_nhwc_out(low, frag, None, 8, 3, 1, 1, 1, True, 3, True, None, b2, 8)
    assert torch.equal(a, b2)
    # K-S, K-R, upsample-add
    img = torch.rand(2, 3, 24, 40, generator=g).to(DEV)
    hw = [torch.randn(*s, generator=g) * 0.3 for s in ((8, 3, 3, 3), (8,), (8, 8, 3, 3), (8,))]
    assert torch.equal(P.conv_stem(img, *hw), ops.conv_stem(img, *hw))
    dh = (2 + torch.rand(2, 1, 12, 20, generator=g)).to(DEV)
    dmin, dmax = torch.tensor([1.0, 1.5], device=DEV), torch.tensor([4.0, 5.0], device=DEV)
    w_low = [torch.randn(*s, generator=g) * 0.3 for s in ((8, 1, 3, 3), (8,), (8, 8, 3, 3), (8,))]
    low = ops.refine_low(dh, dmin, dmax, *w_low)
    assert torch.equal(P.refine_low(dh, dmin, dmax, *w_low), low)
    w_full = [torch.randn(*s, generator=g) * 0.3 for s in ((8, 8, 3, 3), (8,), (8, 3, 3, 3), (8,), (8, 16, 3, 3), (8,), (1, 8, 3, 3))]
    assert torch.equal(P.refine_full(low, img, dh, dmin, dmax, *w_full), ops.refine_full(low, img, dh, dmin, dmax, *w_full))
    ys = _cl(torch.randn(2, 32, 24, 40, generator=g))
    bias = torch.randn(32, generator=g).to(DEV)
    assert torch.equal(P.upsample2x_add(coarse, ys, bias), ops.upsample2x_add(coarse, ys, bias))
    # ragged packs and the *_views forms of K-A
    B, C, G, H, W, D = 2, 32, 8, 24, 40, 8
    maps = [torch.randn(B, C, h, w, generator=g).to(DEV) for h, w in ((24, 40), (40, 24), (13, 21))]
    data, extents = P.pack_nhwc_views(maps)
    pack = ops.pack_nhwc_views(maps)
    assert torch.equal(data, pack.data)
    assert extents.device.type == "cpu" and extents.tolist() == [list(t) for t in zip(pack.offsets, pack.heights, pack.widths)]
    ref = torch.randn(B, H, W, C, generator=g).to(DEV)
    rt = torch.tensor([1, 0, 0, 0, 1, 0, 0, 0, 1, 3.0, -2.0, 0.0]).repeat(3, B, 1).to(DEV)
    depth = (1 + torch.rand(B, D, H, W, generator=g)).to(DEV)
    vw = torch.rand(B, 3, H, W, generator=g).to(DEV)
    assert torch.equal(P.warp_corr_views(ref, data, extents, rt, depth, None, G), ops.warp_corr(ref, pack, rt, depth, G))
    assert torch.equal(P.warp_corr_views(ref, data, extents, rt, depth, vw, G), ops.warp_corr(ref, pack, rt, depth, G, vw))
    net = PatchMatch(num_feature=C, G=G).eval()
    with torch.no_grad():
        for p in net.parameters():
            p.normal_(0, 0.3, generator=g)
    net.refresh_script_heads()
    pw, sim = net.evaluation.pixel_wise_net, net.evaluation.similarity_net
    v0, s0 = P.warp_corr_view_weights_views(ref, data, extents, rt, depth, pw.folded_tensor(), G)
    v1, s1 = ops.warp_corr_view_weights(ref, pack, rt, depth, G, pw.folded(), keep_sims=True)
    assert torch.equal(v0, v1) and torch.equal(s0, s1)
    xs0, xs1 = torch.zeros(B, D, H, W, 2, device=DEV), torch.zeros(B, D, H, W, 2, device=DEV)
    P.warp_corr_score_views_(ref, data, extents, rt, depth, vw, sim.folded_tensor(), G, xs0)
    ops.warp_corr_score(ref, pack, rt, depth, G, vw, sim.folded(), xs=xs1)
    assert torch.equal(xs0, xs1)
    # the cached device copy of a host tensor keeps its values and memory format, and is uploaded once
    wcl = torch.randn(8, 16, 3, 3, generator=g).contiguous(memory_format=torch.channels_last)
    c0, c1 = P.device_copy(wcl, ref), P.device_copy(wcl, ref)
    assert c0.data_ptr() == c1.data_ptr() and torch.equal(c0.cpu(), wcl) and c0.is_contiguous(memory_format=torch.channels_last)


@pytest.mark.gpu
def test_bad_arguments_raise_and_leave_out_untouched():
    P = torch.ops.pmb200
    x = _cl(torch.randn(1, 16, 8, 8))
    frag = ops.pack_conv_filter(torch.randn(16, 16, 3, 3), 3)
    out = torch.full((1, 16, 8, 8), 7.0, device=DEV).contiguous(memory_format=torch.channels_last)
    for call in (lambda: P.conv2d_nhwc_out(x, frag[:-1], None, 16, 3, 1, 1, 1, False, 3, False, None, out, 0),  # filter size
                 lambda: P.conv2d_nhwc_out(x, frag, None, 16, 3, 1, 1, 1, False, 3, False, None, out, 4),  # channel window
                 lambda: P.conv2d_nhwc_out(x, frag, torch.zeros(3), 16, 3, 1, 1, 1, False, 3, False, None, out, 0),  # bias
                 lambda: P.conv2d_nhwc_out(x, frag, None, 16, 3, 2, 1, 1, False, 3, False, None, out, 0),  # out's size
                 lambda: P.conv2d_tc5_out(x, ops.pack_conv_filter_tc5h(torch.randn(16, 16, 3, 3)), None, 16, 3, 2, 1, 1, False, True,
                                          out, 0)):  # halo form at stride 2
        with pytest.raises(RuntimeError):
            call()
        assert bool((out == 7.0).all())
    with pytest.raises(RuntimeError, match="HOST"):
        P.conv_stem(torch.rand(1, 3, 8, 8, device=DEV), *[t.to(DEV) for t in (torch.zeros(8, 3, 3, 3), torch.zeros(8),
                                                                              torch.zeros(8, 8, 3, 3), torch.zeros(8))])
    data, extents = P.pack_nhwc_views([torch.randn(1, 16, 8, 8, device=DEV), torch.randn(1, 16, 4, 6, device=DEV)])
    ref = torch.randn(1, 8, 8, 16, device=DEV)
    rt = torch.zeros(2, 1, 12, device=DEV)
    depth = torch.ones(1, 4, 8, 8, device=DEV)
    bad = extents.clone()
    bad[1, 1] = 100  # past the end of the pack
    with pytest.raises(RuntimeError, match="inside the pack"):
        P.warp_corr_views(ref, data, bad, rt, depth, None, 4)
    bad = extents.clone()
    bad[1, 0] += 1  # not a multiple of 4: the library's own rule
    xs = torch.full((1, 4, 8, 8, 2), 7.0, device=DEV)
    with pytest.raises(RuntimeError):
        P.warp_corr_score_views_(ref, data, bad, rt, depth, torch.ones(1, 2, 8, 8, device=DEV), torch.zeros(289), 4, xs)
    assert bool((xs == 7.0).all())


# ---- deployment --------------------------------------------------------------------------------------------------------------
_FRESH = """
import sys, torch
import patchmatchnet_b200  # registers torch.ops.pmb200
m = torch.jit.load(sys.argv[1], map_location="cpu").cuda()
images, K, E, dmin, dmax = torch.load(sys.argv[2])
with torch.no_grad():
    depth, conf, _ = m([i.cuda() for i in images], K.cuda(), E.cuda(), dmin.cuda(), dmax.cuda())
torch.save((depth.cpu(), conf.cpu()), sys.argv[3])
"""

_LOADER = r"""
#include <dlfcn.h>
#include <torch/script.h>
#include <fstream>
#include <iostream>
#include <iterator>

static std::vector<char> read_all(const char *path) {
    std::ifstream f(path, std::ios::binary);
    return std::vector<char>(std::istreambuf_iterator<char>(f), std::istreambuf_iterator<char>());
}

// usage: loader libpmb200_torch.so module.pt inputs.pt outputs.pt
int main(int argc, char **argv) {
    if (argc != 5) return 2;
    if (!dlopen(argv[1], RTLD_NOW | RTLD_GLOBAL)) {  // registers the pmb200 operators
        std::cerr << dlerror() << "\n";
        return 3;
    }
    torch::jit::Module m = torch::jit::load(argv[2], torch::kCPU);
    m.to(torch::kCUDA);
    m.eval();
    auto in = torch::jit::pickle_load(read_all(argv[3])).toTuple()->elements();
    c10::List<at::Tensor> images;
    for (const auto &im : in[0].toList()) images.push_back(im.get().toTensor().cuda());
    std::vector<torch::jit::IValue> args{images};
    for (size_t i = 1; i < in.size(); ++i) args.push_back(in[i].toTensor().cuda());
    torch::NoGradGuard no_grad;
    auto out = m.forward(args).toTuple()->elements();
    auto bytes = torch::jit::pickle_save(c10::ivalue::Tuple::create({out[0].toTensor().cpu(), out[1].toTensor().cpu()}));
    std::ofstream(argv[4], std::ios::binary).write(bytes.data(), (std::streamsize)bytes.size());
    return 0;
}
"""


def _deployment_case(golden_weights, tmp_path):
    """The golden request, a module scripted with a fixed stage-3 draw (it travels in the archive) and the eager outputs."""
    inp = pm_cases.make_net_inputs(pm_cases.NET_CASE)
    rand = inp["rand48"].to(DEV)
    net = _net(golden_weights, DEV)
    net.patchmatch_3.rand_source = lambda size, device: rand
    net.patchmatch_3.rand_draw = inp["rand48"]
    path = str(tmp_path / "module.pt")
    torch.jit.script(net).save(path)
    depth, conf, _ = _run(net, inp)
    args = (inp["images"], inp["intrinsics"], inp["extrinsics"], inp["depth_min"], inp["depth_max"])
    torch.save(args, str(tmp_path / "inputs.pt"))
    return path, inp, depth.cpu(), conf.cpu()


def _child_env():
    env = dict(os.environ)
    env["PYTHONPATH"] = REPO + os.pathsep + env.get("PYTHONPATH", "")
    return env


@pytest.mark.gpu
def test_archive_runs_in_a_fresh_interpreter_under_data_parallel_and_from_cpp(golden_weights, tmp_path, tf32):
    path, inp, depth, conf = _deployment_case(golden_weights, tmp_path)
    # a fresh interpreter: import the package, torch.jit.load(map_location="cpu").cuda()
    script = tmp_path / "fresh.py"
    script.write_text(_FRESH)
    subprocess.run([sys.executable, str(script), path, str(tmp_path / "inputs.pt"), str(tmp_path / "py_out.pt")], check=True,
                   env=_child_env(), cwd=str(tmp_path))
    d, c = torch.load(str(tmp_path / "py_out.pt"))
    assert d.numpy().tobytes() == depth.numpy().tobytes() and c.numpy().tobytes() == conf.numpy().tobytes()
    # eval.py:38-64: nn.DataParallel(torch.jit.load(...)), model.cuda(), model.eval(), model.forward(...)
    model = torch.nn.DataParallel(torch.jit.load(path))
    model.cuda()
    model.eval()
    with torch.no_grad():
        d, c, _ = model.forward(*_args(inp))
    assert torch.equal(d.cpu(), depth) and torch.equal(c.cpu(), conf)
    # C++: dlopen("libpmb200_torch.so") before torch::jit::load, compiled with the flags of the shim (libtorch_cuda kept in
    # the link although no symbol of it is named: it registers ATen's CUDA backend)
    tdir = os.path.dirname(os.path.abspath(torch.__file__))
    src, exe = tmp_path / "loader.cpp", tmp_path / "loader"
    src.write_text(_LOADER)
    cuda_home = os.environ.get("CUDA_HOME", "/usr/local/cuda")
    subprocess.run(["g++", "-O1", "-std=c++17", f"-D_GLIBCXX_USE_CXX11_ABI={int(torch._C._GLIBCXX_USE_CXX11_ABI)}",
                    f"-I{tdir}/include", f"-I{tdir}/include/torch/csrc/api/include", f"-I{cuda_home}/include", str(src), "-o", str(exe),
                    f"-L{tdir}/lib", "-Wl,--no-as-needed", "-lc10", "-lc10_cuda", "-ltorch_cpu", "-ltorch_cuda", "-ltorch",
                    "-Wl,--as-needed", f"-Wl,-rpath,{tdir}/lib", "-ldl"],
                   check=True)
    subprocess.run([str(exe), _native.TORCH_LIB_PATH, path, str(tmp_path / "inputs.pt"), str(tmp_path / "cpp_out.pt")], check=True)
    d, c = torch.load(str(tmp_path / "cpp_out.pt"))
    assert d.numpy().tobytes() == depth.numpy().tobytes() and c.numpy().tobytes() == conf.numpy().tobytes()


# ---- training end to end -----------------------------------------------------------------------------------------------------
TH, TW = 64, 80


def _write_training_set(root, n_views=3):
    """One plane scene in datasets/mvs.py's layout (pair.txt, cams, depth_gt, images/<light>), as tests/test_gpu_train.py builds its own."""
    from PIL import Image

    from patchmatchnet_b200 import data_io

    base = os.path.join(root, "scan1")
    for sub in ("cams", "depth_gt", os.path.join("images", "0")):
        os.makedirs(os.path.join(base, sub), exist_ok=True)
    with open(os.path.join(base, "pair.txt"), "w") as f:
        f.write(scene_cases.pair_text(scene_cases.all_pairs(n_views, 2)))
    for v, (K, E) in enumerate(scene_cases.cameras(n_views, TH, TW)):
        with open(os.path.join(base, "cams", "%08d_cam.txt" % v), "w") as f:
            f.write(scene_cases.cam_text(K, E))
        depth = plane_depth(K, E, TH, TW, scene_cases.PLANE_N, scene_cases.PLANE_D0).astype(np.float32)
        data_io.save_map(os.path.join(base, "depth_gt", "%08d.pfm" % v), depth)
        Image.fromarray(scene_cases.texture(K, E, TH, TW)).save(os.path.join(base, "images", "0", "%08d.jpg" % v), quality=95)
    for name in ("train.txt", "val.txt"):
        with open(os.path.join(root, name), "w") as f:
            f.write("scan1\n")


@pytest.mark.gpu
def test_trained_module_runs_and_equals_its_checkpoint(tmp_path):
    from patchmatchnet_b200 import reconstruct

    root, out = str(tmp_path / "data"), str(tmp_path / "run")
    _write_training_set(root)
    args = train.parse_args(["--input-folder", root, "--output-folder", out, "--train-list", os.path.join(root, "train.txt"),
                             "--test-list", os.path.join(root, "val.txt"), "--num-views", "2", "--num-light-idx", "1", "--batch-size", "1",
                             "--num-workers", "0", "--image-max-dim", "-1", "--epochs", "2"])
    train.run(args)
    sm = torch.jit.load(os.path.join(out, "module_000001.pt"), map_location="cpu").cuda()
    ck = torch.load(os.path.join(out, "params_000001.ckpt"), map_location="cpu")
    with reconstruct.precision(False):  # what train froze the archive under (its default, no --tf32)
        net = train.build_network(train.parse_args([]))
        load_reference_state(net, ck["model"])
        net = net.to(DEV).eval()
        inp = pm_cases.make_net_inputs(dict(B=1, n_views=3, H=TH, W=TW, seed=9))
        rand = inp["rand48"].to(DEV)
        net.patchmatch_3.rand_source = lambda size, device: rand
        sm.patchmatch_3.rand_draw = rand
        _assert_same(_run(net, inp), _run(sm, inp))
