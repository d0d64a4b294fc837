"""CPU/PyTorch oracle for PatchmatchNet's learned-PatchMatch hot path.

TEST INFRASTRUCTURE ONLY.  Nothing under ``patchmatchnet_b200/`` imports this
package; only ``tests/``, ``__graft_entry__.smoke()`` and ``bench.py``'s
``cpu_baseline`` / ``--impl reference`` legs may.  The product path has no CPU
fallback and never routes through here.

What it is: a functional restatement (plain torch fp32 ops, runs on CPU or any
torch device) of the algorithm in the reference's ``models/patchmatch.py`` and
``models/module.py:130-181``.  The floating-point arithmetic of the path lives
in PyTorch ATen (``grid_sampler_2d``, ``linalg_inv``, ``sort``, conv/BN) which
is a third-party dependency of the reference (``requirements.txt:1`` pins no
version; the installed wheel is torch 2.11.0+cu128) -- the oracle calls the
same ATen entry points in the same order so that, on the same device, it is
bit-identical to the reference.

Parity pin: the reference ships no tests or golden vectors ("parity unpinned"
by the reference's own tests, SURVEY.md 8c).  The oracle is pinned instead
against what the UNMODIFIED reference computed on the same seeded inputs,
recorded by ``tests/golden/make_golden.py`` and
``tests/golden/make_reference_vectors.py`` into ``tests/golden/*.pt``
(``tests/test_oracle_vs_reference.py``: max-abs diff == 0 on CPU;
``tests/test_golden.py``).

Every function cites the reference lines it restates.
"""
from __future__ import annotations

from typing import Callable, List, Optional, Sequence, Tuple

import torch
import torch.nn as nn
import torch.nn.functional as F

Tensor = torch.Tensor

# --------------------------------------------------------------------------
# a1: homography warp (models/module.py:130-181)
# --------------------------------------------------------------------------


def relative_projection(src_proj: Tensor, ref_proj: Tensor) -> Tuple[Tensor, Tensor]:
    """rot [B,3,3], trans [B,3,1] of src_proj @ inv(ref_proj) (module.py:148-150)."""
    rel = torch.matmul(src_proj, torch.inverse(ref_proj))
    return rel[:, :3, :3], rel[:, :3, 3:4]


def homography_warp(src_fea: Tensor, src_proj: Tensor, ref_proj: Tensor, depth: Tensor) -> Tensor:
    """Warp ``src_fea [B,C,Hs,Ws]`` to every depth hypothesis ``depth [B,D,H,W]``.

    Returns ``[B,C,D,H,W]``.  module.py:144-181: pixel (x,y,1) is rotated, scaled
    by depth, translated; points with z <= 1e-3 are sent to (W,H,1) so that all
    four taps fall outside and zero padding returns 0; the rest is a bilinear
    lookup at (x/z, y/z) in pixel units (normalise + align_corners=True cancel).
    """
    B, D, H, W = depth.shape
    C = src_fea.shape[1]
    dev = src_fea.device
    with torch.no_grad():
        rot, trans = relative_projection(src_proj, ref_proj)
        ys, xs = torch.meshgrid(
            torch.arange(0, H, dtype=torch.float32, device=dev),
            torch.arange(0, W, dtype=torch.float32, device=dev),
            indexing="ij",
        )
        ys, xs = ys.reshape(H * W), xs.reshape(H * W)
        pix = torch.stack((xs, ys, torch.ones_like(xs))).unsqueeze(0).repeat(B, 1, 1)  # [B,3,HW]
        ray = torch.matmul(rot, pix)  # [B,3,HW]
        pts = ray.unsqueeze(2).repeat(1, 1, D, 1) * depth.view(B, 1, D, H * W)
        pts = pts + trans.view(B, 3, 1, 1)  # [B,3,D,HW]
        behind = pts[:, 2:] <= 1e-3
        pts[:, 0:1][behind] = float(W)
        pts[:, 1:2][behind] = float(H)
        pts[:, 2:3][behind] = 1.0
        uv = pts[:, :2] / pts[:, 2:3]
        gx = uv[:, 0] / ((W - 1) / 2) - 1
        gy = uv[:, 1] / ((H - 1) / 2) - 1
        grid = torch.stack((gx, gy), dim=3)  # [B,D,HW,2]
    out = F.grid_sample(
        src_fea, grid.view(B, D * H, W, 2), mode="bilinear", padding_mode="zeros", align_corners=True
    )
    return out.view(B, C, D, H, W)


# --------------------------------------------------------------------------
# a2: group-wise correlation (models/patchmatch.py:193, 199-203)
# --------------------------------------------------------------------------


def groupwise_correlation(warped: Tensor, ref_fea: Tensor, groups: int) -> Tensor:
    """mean over the C/G channels of each group of warped*ref -> [B,G,D,H,W]."""
    B, C, D, H, W = warped.shape
    r = ref_fea.view(B, groups, C // groups, 1, H, W)
    return (warped.view(B, groups, C // groups, D, H, W) * r).mean(2)


# --------------------------------------------------------------------------
# a7: neighbour tables and sampling grid (models/patchmatch.py:314-426)
# --------------------------------------------------------------------------


def neighbour_table(kind: str, count: int, dilation: int) -> List[Tuple[int, int]]:
    """Fixed (dy, dx) offsets.  patchmatch.py:331-392.

    propagation: 4 / 8 / 16 neighbours at +-dilation (16 = ring + doubled ring);
    evaluation : 9 / 17 neighbours at +-(dilation-1) (17 = 3x3 + doubled ring w/o centre).
    Entry order is (dy, dx): patchmatch.py:409 unpacks ``offset_y, offset_x``.
    """
    if kind == "propagation":
        d = dilation
        if count == 4:
            return [(-d, 0), (0, -d), (0, d), (d, 0)]
        ring = [(-d, -d), (-d, 0), (-d, d), (0, -d), (0, d), (d, -d), (d, 0), (d, d)]
        if count == 8:
            return ring
        if count == 16:
            return ring + [(2 * a, 2 * b) for a, b in ring]
        raise NotImplementedError
    if kind == "evaluation":
        d = dilation - 1
        box = [(-d, -d), (-d, 0), (-d, d), (0, -d), (0, 0), (0, d), (d, -d), (d, 0), (d, d)]
        if count == 9:
            return box
        if count == 17:
            return box + [(2 * a, 2 * b) for a, b in box if a != 0 or b != 0]
        raise NotImplementedError
    raise NotImplementedError


def sampling_grid(table: Sequence[Tuple[int, int]], learned: Tensor, H: int, W: int) -> Tensor:
    """Normalised sampling grid [B, K*H, W, 2] from ``learned [B,2K,H*W]``.

    patchmatch.py:396-426.  learned[:, 2k] is the x offset, learned[:, 2k+1] the y
    offset (:410-411).  The normalisation is the align_corners=True one (:420-421)
    although the grids are consumed with align_corners=False -- reproduced as is.
    """
    B = learned.shape[0]
    dev = learned.device
    with torch.no_grad():
        ys, xs = torch.meshgrid(
            torch.arange(0, H, dtype=torch.float32, device=dev),
            torch.arange(0, W, dtype=torch.float32, device=dev),
            indexing="ij",
        )
        base = torch.stack((xs.reshape(H * W), ys.reshape(H * W))).unsqueeze(0).repeat(B, 1, 1)  # [B,2,HW]
    pos = []
    for k, (dy, dx) in enumerate(table):
        ox = dx + learned[:, 2 * k, :].unsqueeze(1)
        oy = dy + learned[:, 2 * k + 1, :].unsqueeze(1)
        pos.append((base + torch.cat((ox, oy), dim=1)).unsqueeze(2))
    pos = torch.cat(pos, dim=2)  # [B,2,K,HW]
    gx = pos[:, 0] / ((W - 1) / 2) - 1
    gy = pos[:, 1] / ((H - 1) / 2) - 1
    return torch.stack((gx, gy), dim=3).view(B, len(table) * H, W, 2)


def _border_sample(x: Tensor, grid: Tensor) -> Tensor:
    """The lookup used by a6/a8/a10/a11: bilinear, border padding, align_corners=False."""
    return F.grid_sample(x, grid, mode="bilinear", padding_mode="border", align_corners=False)


# --------------------------------------------------------------------------
# a9: hypothesis initialisation (models/patchmatch.py:17-94)
# --------------------------------------------------------------------------

NUM_RANDOM_BINS = 48  # hard-coded in patchmatch.py:59


def init_hypotheses(
    depth_min: Tensor,
    depth_max: Tensor,
    H: int,
    W: int,
    interval_scale: float,
    num_sample: int,
    depth: Tensor,
    device: torch.device,
    rand_source: Optional[Callable] = None,
) -> Tensor:
    """[B,48,H,W] stratified random inverse-depth samples when ``depth`` is empty
    (patchmatch.py:56-71), ``depth`` itself when num_sample == 1 (:73-74), else
    num_sample local perturbations in inverse depth, clamped to the range (:75-94)."""
    B = depth_min.size(0)
    inv_min = 1.0 / depth_min
    inv_max = 1.0 / depth_max
    if depth.numel() == 0:
        n = NUM_RANDOM_BINS
        draw = rand_source if rand_source is not None else torch.rand
        u = draw(size=(B, n, H, W), device=device)
        s = u + torch.arange(start=0, end=n, step=1, device=device).view(1, n, 1, 1)
        s = inv_max.view(B, 1, 1, 1) + s / n * (inv_min.view(B, 1, 1, 1) - inv_max.view(B, 1, 1, 1))
        return 1.0 / s
    if num_sample == 1:
        return depth.detach()
    k = (
        torch.arange(-num_sample // 2, num_sample // 2, 1, device=device)
        .view(1, num_sample, 1, 1)
        .repeat(B, 1, H, W)
        .float()
    )
    step = ((inv_min - inv_max) * interval_scale).view(B, 1, 1, 1)
    s = 1.0 / depth.detach() + step * k
    rows = [torch.clamp(s[b], min=inv_max[b], max=inv_min[b]).unsqueeze(0) for b in range(B)]
    return 1.0 / torch.cat(rows, dim=0)


# --------------------------------------------------------------------------
# a8: adaptive propagation (models/patchmatch.py:97-124)
# --------------------------------------------------------------------------


def propagate(depth_sample: Tensor, grid: Tensor) -> Tensor:
    """Gather the centre hypothesis D//2 at the Kp neighbours, append, sort ascending."""
    B, D, H, W = depth_sample.shape
    K = grid.size(1) // H
    centre = depth_sample[:, D // 2, :, :].unsqueeze(1)
    got = _border_sample(centre, grid).view(B, K, H, W)
    return torch.sort(torch.cat((depth_sample, got), dim=1), dim=1)[0]


# --------------------------------------------------------------------------
# a10: depth-similarity weight (models/patchmatch.py:627-669)
# --------------------------------------------------------------------------


def depth_similarity_weight(
    depth_sample: Tensor, depth_min: Tensor, depth_max: Tensor, grid: Tensor, interval_scale: float, neighbours: int
) -> Tensor:
    B, D, H, W = depth_sample.shape
    inv_min = 1.0 / depth_min
    inv_max = 1.0 / depth_max
    x = 1.0 / depth_sample
    x = (x - inv_max.view(B, 1, 1, 1)) / (inv_min - inv_max).view(B, 1, 1, 1)
    x1 = _border_sample(x, grid).view(B, D, neighbours, H, W)
    x1 = torch.abs(x1 - x.unsqueeze(2)) / interval_scale
    return torch.sigmoid(4.0 - 2.0 * x1.clamp(min=0, max=4)).detach()


# --------------------------------------------------------------------------
# learned 1x1x1 heads (ConvBnReLU3D: models/module.py:43-72)
# --------------------------------------------------------------------------


class _PointwiseBlock(nn.Module):
    """conv3d(1x1x1, no bias) + BatchNorm3d + ReLU, parameter names ``conv`` / ``bn``."""

    def __init__(self, cin: int, cout: int) -> None:
        super().__init__()
        self.conv = nn.Conv3d(cin, cout, 1, stride=1, padding=0, dilation=1, bias=False)
        self.bn = nn.BatchNorm3d(cout)

    def forward(self, x: Tensor) -> Tensor:
        return F.relu(self.bn(self.conv(x)), inplace=True)


class _ViewWeightHead(nn.Module):
    """a4 PixelwiseNet, patchmatch.py:672-702."""

    def __init__(self, G: int) -> None:
        super().__init__()
        self.conv0 = _PointwiseBlock(G, 16)
        self.conv1 = _PointwiseBlock(16, 8)
        self.conv2 = nn.Conv3d(8, 1, 1, stride=1, padding=0)

    def forward(self, sim: Tensor) -> Tensor:
        y = torch.sigmoid(self.conv2(self.conv1(self.conv0(sim))).squeeze(1))
        return torch.max(y, dim=1)[0].unsqueeze(1)


class _ScoreHead(nn.Module):
    """a6 SimilarityNet, patchmatch.py:532-577."""

    def __init__(self, G: int) -> None:
        super().__init__()
        self.conv0 = _PointwiseBlock(G, 16)
        self.conv1 = _PointwiseBlock(16, 8)
        self.similarity = nn.Conv3d(8, 1, 1, stride=1, padding=0)

    def raw_score(self, sim: Tensor) -> Tensor:
        return self.similarity(self.conv1(self.conv0(sim))).squeeze(1)  # [B,D,H,W]

    def forward(self, sim: Tensor, grid: Tensor, weight: Tensor) -> Tensor:
        B, _, D, H, W = sim.shape
        K = grid.size(1) // H
        s = _border_sample(self.raw_score(sim), grid).view(B, D, K, H, W)
        return torch.sum(s * weight, dim=2)


class _FeatureWeightHead(nn.Module):
    """a11 FeatureWeightNet, patchmatch.py:580-624."""

    def __init__(self, neighbours: int, G: int) -> None:
        super().__init__()
        self.neighbours = neighbours
        self.G = G
        self.conv0 = _PointwiseBlock(G, 16)
        self.conv1 = _PointwiseBlock(16, 8)
        self.similarity = nn.Conv3d(8, 1, 1, stride=1, padding=0)

    def neighbour_correlation(self, ref_fea: Tensor, grid: Tensor) -> Tensor:
        B, C, H, W = ref_fea.shape
        g = _border_sample(ref_fea, grid).view(B, self.G, C // self.G, self.neighbours, H, W)
        c = ref_fea.view(B, self.G, C // self.G, H, W).unsqueeze(3)
        return (g * c).mean(2)  # [B,G,K,H,W]

    def forward(self, ref_fea: Tensor, grid: Tensor) -> Tensor:
        corr = self.neighbour_correlation(ref_fea, grid)
        return torch.sigmoid(self.similarity(self.conv1(self.conv0(corr))).squeeze(1))


# --------------------------------------------------------------------------
# a3/a5: evaluation (models/patchmatch.py:145-239)
# --------------------------------------------------------------------------


class _Evaluation(nn.Module):
    def __init__(self, G: int) -> None:
        super().__init__()
        self.G = G
        self.pixel_wise_net = _ViewWeightHead(G)
        self.similarity_net = _ScoreHead(G)

    def aggregate_views(
        self,
        ref_fea: Tensor,
        src_feas: Sequence[Tensor],
        ref_proj: Tensor,
        src_projs: Sequence[Tensor],
        depth_sample: Tensor,
        view_weights: Tensor,
    ) -> Tuple[Tensor, Tensor]:
        """patchmatch.py:191-217,223-224 -> (similarity [B,G,D,H,W], view_weights [B,V,H,W])."""
        B, C, H, W = ref_fea.shape
        D = depth_sample.size(1)
        dev = ref_fea.device
        assert len(src_feas) == len(src_projs), "Patchmatch Evaluation: Different number of images and projection matrices"
        have_w = view_weights.numel() != 0
        if have_w:
            assert len(src_feas) == view_weights.size(1), "Patchmatch Evaluation: Different number of images and view weights"
        wsum = 1e-5 * torch.ones((B, 1, 1, H, W), dtype=torch.float32, device=dev)
        ssum = torch.zeros((B, self.G, D, H, W), dtype=torch.float32, device=dev)
        fresh = []
        for v, (sf, sp) in enumerate(zip(src_feas, src_projs)):
            sim = groupwise_correlation(homography_warp(sf, sp, ref_proj, depth_sample), ref_fea, self.G)
            if have_w:
                vw = view_weights[:, v].unsqueeze(1)
            else:
                vw = self.pixel_wise_net(sim)
                fresh.append(vw)
            ssum += sim * vw.unsqueeze(1)
            wsum += vw.unsqueeze(1)
        sim = ssum.div_(wsum)
        if not have_w:
            view_weights = torch.cat(fresh, dim=1)
        return sim, view_weights

    @staticmethod
    def regress(depth_sample: Tensor, prob: Tensor, is_inverse: bool) -> Tensor:
        """patchmatch.py:226-237."""
        D = depth_sample.size(1)
        if is_inverse:
            idx = torch.arange(0, D, 1, device=prob.device).view(1, D, 1, 1)
            idx = torch.sum(idx * prob, dim=1)
            inv_hi = 1.0 / depth_sample[:, -1, :, :]
            inv_lo = 1.0 / depth_sample[:, 0, :, :]
            return 1.0 / (inv_lo + idx / (D - 1) * (inv_hi - inv_lo))
        return torch.sum(depth_sample * prob, dim=1)

    def forward(self, ref_fea, src_feas, ref_proj, src_projs, depth_sample, grid, weight, view_weights, is_inverse):
        sim, view_weights = self.aggregate_views(ref_fea, src_feas, ref_proj, src_projs, depth_sample, view_weights)
        score = self.similarity_net(sim, grid, weight)
        prob = torch.exp(F.log_softmax(score, dim=1))
        return self.regress(depth_sample, prob, is_inverse), prob, view_weights.detach()


# --------------------------------------------------------------------------
# a12/a13: the PatchMatch module (models/patchmatch.py:242-529)
# --------------------------------------------------------------------------


class PatchMatchOracle(nn.Module):
    """Same constructor, forward signature, parameter names and shapes as the
    reference ``PatchMatch`` (patchmatch.py:245-312, :428-529) so the reference's
    state dicts load with all keys matched."""

    def __init__(
        self,
        propagation_out_range: int = 2,
        patchmatch_iteration: int = 2,
        patchmatch_num_sample: int = 16,
        patchmatch_interval_scale: float = 0.025,
        num_feature: int = 64,
        G: int = 8,
        propagate_neighbors: int = 16,
        evaluate_neighbors: int = 9,
        stage: int = 3,
    ) -> None:
        super().__init__()
        self.patchmatch_iteration = patchmatch_iteration
        self.patchmatch_interval_scale = patchmatch_interval_scale
        self.patchmatch_num_sample = patchmatch_num_sample
        self.G = G
        self.stage = stage
        self.dilation = propagation_out_range
        self.propagate_neighbors = propagate_neighbors
        self.evaluate_neighbors = evaluate_neighbors
        self.rand_source: Optional[Callable] = None  # tests inject a shared U[0,1) draw here
        self.evaluation = _Evaluation(G)
        self.propa_conv = nn.Conv2d(
            num_feature, max(2 * propagate_neighbors, 1), 3, stride=1,
            padding=self.dilation, dilation=self.dilation, bias=True,
        )
        self.eval_conv = nn.Conv2d(
            num_feature, 2 * evaluate_neighbors, 3, stride=1,
            padding=self.dilation, dilation=self.dilation, bias=True,
        )
        for conv in (self.propa_conv, self.eval_conv):  # patchmatch.py:297-298, 310-311
            nn.init.constant_(conv.weight, 0.0)
            nn.init.constant_(conv.bias, 0.0)
        self.feature_weight_net = _FeatureWeightHead(evaluate_neighbors, G)

    def forward(
        self,
        ref_feature: Tensor,
        src_features: List[Tensor],
        ref_proj: Tensor,
        src_projs: List[Tensor],
        depth_min: Tensor,
        depth_max: Tensor,
        depth: Tensor,
        view_weights: Tensor,
    ) -> Tuple[List[Tensor], Tensor, Tensor]:
        dev = ref_feature.device
        B, _, H, W = ref_feature.shape
        Kp, Ke = self.propagate_neighbors, self.evaluate_neighbors

        propa_grid = torch.empty(0, device=dev)
        if Kp > 0 and not (self.stage == 1 and self.patchmatch_iteration == 1):  # :465
            off = self.propa_conv(ref_feature).view(B, 2 * Kp, H * W)
            propa_grid = sampling_grid(neighbour_table("propagation", Kp, self.dilation), off, H, W)
        off = self.eval_conv(ref_feature).view(B, 2 * Ke, H * W)  # :471
        eval_grid = sampling_grid(neighbour_table("evaluation", Ke, self.dilation), off, H, W)
        feature_weight = self.feature_weight_net(ref_feature.detach(), eval_grid)  # :475

        sample = depth
        prob = torch.empty(0, device=dev)
        outs: List[Tensor] = []
        for it in range(1, self.patchmatch_iteration + 1):
            last_of_stage1 = self.stage == 1 and it == self.patchmatch_iteration  # :482
            sample = init_hypotheses(
                depth_min, depth_max, H, W, self.patchmatch_interval_scale,
                self.patchmatch_num_sample, sample, dev, self.rand_source,
            )
            if Kp > 0 and not last_of_stage1:  # :497
                sample = propagate(sample, propa_grid)
            w = depth_similarity_weight(
                sample.detach(), depth_min, depth_max, eval_grid.detach(), self.patchmatch_interval_scale, Ke
            ) * feature_weight.unsqueeze(1)
            w = w / torch.sum(w, dim=2).unsqueeze(2)  # :510
            sample, prob, view_weights = self.evaluation(
                ref_feature, src_features, ref_proj, src_projs, sample, eval_grid, w, view_weights, last_of_stage1
            )
            sample = sample.unsqueeze(1)
            outs.append(sample)
        return outs, prob, view_weights
