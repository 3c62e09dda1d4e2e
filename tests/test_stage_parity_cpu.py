"""CPU side of the stage tests (tests/test_stage_parity_gpu.py): the clouds reach the occupancies they are built for
(the oracle's voxel indices), and the TF32 operand models are the bit-level operations they claim to be."""
import numpy as np
import pytest
import torch

from tests import stage_ref as SR


@pytest.mark.parametrize("K,N,r", [(127, 2048, 32), (128, 2048, 32), (129, 2048, 32), (256, 2048, 32), (127, 1024, 16),
                                   (128, 1024, 16), (129, 1024, 16), (256, 1024, 16), (129, 700, 32), (256, 4096, 32),
                                   (127, 256, 8), (129, 256, 8)])
def test_sites_cloud_occupancy(K, N, r):
    c = SR.sites_cloud(K, N, r, seed=K + N + r)
    assert c.shape == (3, N)
    assert SR.occupancy(c[None], r) == [K]


@pytest.mark.parametrize("N,r", [(2048, 32), (4096, 32), (1024, 16), (500, 13), (64, 8)])
def test_clustered_cloud_occupancy(N, r):
    c = SR.clustered_cloud(N)
    ids = SR.voxel_ids(c[None], r)[0]
    vals, counts = torch.unique(ids, return_counts=True)
    assert len(vals) == 7 and int(counts.max()) == N - 6
    xyz = torch.stack([ids[-6:] // (r * r), ids[-6:] // r % r, ids[-6:] % r], 1)
    for k in range(6):                                        # each extreme point sits on a face of the grid
        assert int(xyz[k, k // 2]) == (r - 1 if k % 2 == 0 else 0)


def test_gaussian_cloud_is_spread():
    occ = SR.occupancy(SR.gaussian_cloud(3, 2048)[None], 32)[0]
    assert 1000 < occ <= 2048


def _tf32_bits_reference(x, mode):
    """Rounding of float32 values to 10 mantissa bits, computed from frexp in float64."""
    x = x.numpy().astype(np.float64)
    m, e = np.frexp(np.abs(x))                  # |x| = m * 2^e, m in [0.5, 1)
    q = m * 2.0 ** 11                           # 11 significant bits: 1 implicit + 10
    q = np.floor(q) if mode == "trunc" else np.floor(q + 0.5)
    return torch.from_numpy((np.sign(x) * np.ldexp(q / 2.0 ** 11, e)).astype(np.float32))


def test_tf32_operand_models_match_their_definitions():
    g = torch.Generator().manual_seed(5)
    x = torch.cat([torch.randn(100000, generator=g) * 10 ** torch.randint(-6, 6, (100000,), generator=g).float(),
                   torch.tensor([1.0, -1.0, 1.0 + 2 ** -11, -(1.0 + 2 ** -11), 1.0 + 3 * 2 ** -11, 1.5 - 2 ** -23, 0.0])])
    assert torch.equal(SR.tf32_trunc(x), _tf32_bits_reference(x, "trunc"))
    assert torch.equal(SR.tf32_rna(x), _tf32_bits_reference(x, "rna"))
    # ties go away from zero; truncation goes toward zero
    assert SR.tf32_rna(torch.tensor([1.0 + 2 ** -11, -(1.0 + 2 ** -11)])).tolist() == [1.0 + 2 ** -10, -(1.0 + 2 ** -10)]
    assert SR.tf32_trunc(torch.tensor([1.0 + 2 ** -10 - 2 ** -23])).tolist() == [1.0]


def test_scatter_grid_model_is_the_fused_multiply_add_chain():
    """scatter_grid = f0 * (1/n), then fma(f_k, 1/n, acc) over the voxel's points in ascending order."""
    g = torch.Generator().manual_seed(6)
    feats = torch.randn(1, 3, 50, generator=g)
    ids = torch.randint(0, 4, (1, 50), generator=g)
    grid = SR.scatter_grid(feats, ids, 2).view(3, 8)
    for v in range(8):
        pts = (ids[0] == v).nonzero().flatten().tolist()
        for c in range(3):
            if not pts:
                assert grid[c, v] == 0
                continue
            inv = np.float32(1.0) / np.float32(len(pts))
            acc = np.float32(feats[0, c, pts[0]].item()) * inv
            for k in pts[1:]:
                acc = np.float32(np.float64(feats[0, c, k].item()) * np.float64(inv) + np.float64(acc))
            assert grid[c, v].item() == acc


# ---------------------------------------------------------------------------------------------------------------------
# second half of a PVConv and the linear attention (tests/test_pvconv_tail_stage_gpu.py, test_attention_stage_gpu.py):
# the float64 references, chained with the TF32 models switched off, restate the fp32 oracle
# ---------------------------------------------------------------------------------------------------------------------
def _cfg():
    from lion_b200.config import default_prior_cfg
    return default_prior_cfg()


def _sd(mod, seed):
    from tests.synth import synth_state_dict
    return synth_state_dict({k: list(v.shape) for k, v in mod.state_dict().items()}, seed)


def _gn(sd, p, style):
    fb = style.double() @ sd[p + "emd.weight"].double().T + sd[p + "emd.bias"].double()
    return sd[p + "norm.weight"].double(), sd[p + "norm.bias"].double(), fb


def _rel(a, b):
    return ((a.double() - b.double()).abs().max() / b.double().abs().max()).item()


@pytest.mark.parametrize("cin,cout,r,N,attn", [(4, 32, 6, 150, False), (16, 32, 5, 90, True), (20, 40, 5, 100, False)])
def test_pvconv_stage_references_restate_the_oracle(cin, cout, r, N, attn):
    from lion_b200.models.pvcnn2_ada import PVConv
    from oracle import net as ON
    from oracle import point_ops as OP
    sd = _sd(PVConv(cin, cout, 3, r, with_se=True, attention=attn, cfg=_cfg()), 7)
    B = 2
    feats, style = torch.randn(B, cin, N, generator=torch.Generator().manual_seed(1)), torch.randn(B, 128)
    coords = torch.randn(B, 3, N, generator=torch.Generator().manual_seed(2)) * 0.4
    V = float(r ** 3)
    raw1 = SR.conv1_reference(feats, coords, sd["voxel_layers.0.weight"], sd["voxel_layers.0.bias"], r, tc=False)
    s1, t1 = SR.fold_affine(raw1.sum((2, 3, 4)), (raw1 * raw1).sum((2, 3, 4)), *_gn(sd, "voxel_layers.1.", style), V)
    act = SR.act_grid(raw1.float(), s1.float(), t1.float(), rna=False)[:, :, 1:-1, 1:-1, 1:-1]
    raw2 = SR.conv3x3x3_f64(act.double(), sd["voxel_layers.4.weight"].double(), sd["voxel_layers.4.bias"].double())
    s2, t2 = SR.fold_se(raw2.sum((2, 3, 4)), (raw2 * raw2).sum((2, 3, 4)), *_gn(sd, "voxel_layers.5.", style), V,
                        sd["voxel_layers.6.fc.0.weight"], sd["voxel_layers.6.fc.2.weight"])
    rawp = SR.point_conv(feats, sd["point_features.layers.0.weight"], sd["point_features.layers.0.bias"], tc=False)
    sp, tp = SR.fold_affine(rawp.sum(2), (rawp * rawp).sum(2), *_gn(sd, "point_features.layers.1.", style), float(N))
    nc, _ = OP.voxel_coords_cuda_order(coords, r)
    out = SR.devox_fuse(raw2, s2, t2, nc, rawp, sp, tp)
    if attn:
        qkv = SR.attn_qkv(out.float(), sd["attn.to_qkv.weight"], tc=False)
        out = SR.attn_out(SR.attn_core(qkv, 4).float(), sd["attn.to_out.weight"], sd["attn.to_out.bias"], tc=False)
    ref = ON.pvconv(sd, "", dict(kind="pvconv", cin=cin, cout=cout, r=r, attn=attn), feats, coords, style)
    assert _rel(out, ref) < 2e-5


@pytest.mark.parametrize("C,heads,N", [(64, 4, 129), (128, 8, 300)])
def test_attention_references_restate_the_oracle(C, heads, N):
    from lion_b200.models.pvcnn2_ada import LinearAttention
    from oracle import net as ON
    sd = _sd(LinearAttention(C, heads), 8)
    x = torch.randn(2, C, N, generator=torch.Generator().manual_seed(3))
    qkv = SR.attn_qkv(x, sd["to_qkv.weight"], tc=False)
    out = SR.attn_out(SR.attn_core(qkv, heads).float(), sd["to_out.weight"], sd["to_out.bias"], tc=False)
    assert _rel(out, ON.linear_attention(sd, "", x, heads)) < 1e-5


def test_trilinear_reference_restates_the_oracle():
    """Including points on the grid's faces and at integer coordinates, where the high corners weigh 0."""
    from oracle import point_ops as OP
    r, N = 6, 400
    g = torch.Generator().manual_seed(4)
    grid = torch.randn(2, 5, r, r, r, generator=g)
    nc = torch.rand(2, 3, N, generator=g) * (r - 1)
    nc[:, :, :50] = torch.randint(0, r, (2, 3, 50), generator=g).float()
    nc[:, 0, 50:60] = r - 1
    got = SR.trilinear_f64(grid.double(), nc, r)
    assert _rel(got, OP.trilinear_devoxelize(grid, nc, r)) < 1e-6
    assert torch.equal(got[:, :, :50], grid.double().reshape(2, 5, -1).gather(
        2, ((nc[:, 0, :50] * r + nc[:, 1, :50]) * r + nc[:, 2, :50]).long()[:, None].expand(2, 5, 50)))


def test_act_grid_model_matches_its_definition():
    """act_grid = rna(float32(swish(float32(x * scale + shift)))) inside, 0 on every halo position."""
    g = torch.Generator().manual_seed(9)
    B, C, r = 2, 3, 3
    raw = torch.randn(B, C, r, r, r, generator=g) * 4
    s, t = torch.randn(B, C, generator=g), torch.randn(B, C, generator=g)
    got = SR.act_grid(raw, s, t)
    assert got.shape == (B, C, r + 2, r + 2, r + 2) and got.dtype == torch.float32
    inner = got[:, :, 1:-1, 1:-1, 1:-1]
    halo = got.clone()
    halo[:, :, 1:-1, 1:-1, 1:-1] = 0
    assert (halo == 0).all()
    for b in range(B):
        for c in range(C):
            for i, v in enumerate(raw[b, c].flatten().tolist()):
                a = np.float32(np.float64(v) * np.float64(s[b, c].item()) + np.float64(t[b, c].item()))
                y = np.float32(np.float64(a) / (1.0 + np.exp(-np.float64(a))))
                want = _tf32_bits_reference(torch.tensor([y]), "rna")[0].item()
                assert inner[b, c].flatten()[i].item() == want
