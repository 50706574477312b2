"""The tf32 weight split image of the tensor-core GEMM (geob200_split_tf32) against a numpy emulation of its rounding."""
import numpy as np
import pytest
import torch

from geotransformer_b200 import functional as GF


def _tf32_rna(w):
    """round-to-nearest tf32, ties away from zero, on the bit pattern: add half an ulp of the 10-bit mantissa to the magnitude
    and clear the low 13 bits (carries into the exponent give the next binade or inf, as the hardware conversion does)"""
    u = w.view(np.uint32)
    hi = ((u + np.uint32(0x1000)) & np.uint32(0xFFFFE000)).view(np.float32)
    return np.where(np.isnan(w), np.float32(np.nan), hi).astype(np.float32)


def _special_values():
    f32 = np.float32
    tiny = np.finfo(f32).tiny
    vals = [0.0, -0.0, np.inf, -np.inf, np.nan, 1.0, -1.0, np.finfo(f32).max, -np.finfo(f32).max, tiny, -tiny,
            tiny / 2, -tiny / 3, np.float32(1e-45), np.float32(-1e-45), 3.0e-39, 65504.0, 1e30, -1e-30]
    # exact ties: mantissa low 13 bits = 0x1000 (halfway), with even and odd retained mantissas, both signs
    bits = [0x3F801000, 0x3F803000, 0xBF801000, 0xBF803000, 0x00001000, 0x00003000, 0x7F7FF000, 0x3F800FFF, 0x3F801001]
    return np.concatenate([np.array(vals, dtype=f32), np.array(bits, dtype=np.uint32).view(f32)])


@pytest.mark.gpu
@pytest.mark.parametrize('n,k,ld', [(64, 32, 32), (48, 100, 100), (256, 768, 800), (7, 28, 40)])
def test_split_image_matches_numpy(n, k, ld):
    rng = np.random.default_rng(n * 1000 + k)
    full = (rng.standard_normal((n, ld)) * np.exp2(rng.integers(-140, 120, (n, ld)))).astype(np.float32)
    sp = _special_values()
    full.reshape(-1)[:sp.size] = sp
    w = torch.from_numpy(full).cuda()[:, :k]
    img = GF.split_tf32(w).cpu().numpy()
    assert img.shape == (2 * n, k)
    x = full[:, :k]
    hi = _tf32_rna(x)
    with np.errstate(invalid='ignore', over='ignore'):
        lo = (x - hi).astype(np.float32)
    for got, want in ((img[:n], hi), (img[n:], lo)):
        nan = np.isnan(want)
        assert np.array_equal(np.isnan(got), nan)
        assert np.array_equal(got[~nan].view(np.uint32), want[~nan].view(np.uint32))
    assert np.all((img[:n].view(np.uint32) & np.uint32(0x1FFF))[~np.isnan(hi)] == 0)


@pytest.mark.gpu
def test_native_images_follow_load_state_dict():
    """The native drivers read cached split images of the weights: after load_state_dict with new weights they must give
    what the module path (which splits on every call) gives with the new weights, bit for bit."""
    from geotransformer_b200.config import make_cfg
    from geotransformer_b200.model import create_model, enable_native
    from geotransformer_b200.synth import make_pair
    from geotransformer_b200.utils.data import registration_collate_fn_stack_mode
    from geotransformer_b200.weights import synthetic_state_dict

    cfg = make_cfg('3dmatch')
    model = create_model(cfg)
    model.load_state_dict(synthetic_state_dict(model, 7351), strict=True)
    model = model.cuda().eval()
    pair = make_pair('demo2k', 0)
    dd = {k: pair[k] for k in ('ref_points', 'src_points', 'ref_feats', 'src_feats', 'transform')}
    data = registration_collate_fn_stack_mode([dd], cfg.backbone.num_stages, cfg.backbone.init_voxel_size,
                                              cfg.backbone.init_radius, cfg.neighbor_limits)
    enable_native(model)
    before = model(data)['ref_feats_c'].clone()
    model.load_state_dict(synthetic_state_dict(model, 1234), strict=True)
    native = model(data)['ref_feats_c'].clone()
    keep, model._native = model._native, None
    module = model(data)['ref_feats_c'].clone()
    model._native = keep
    torch.cuda.synchronize()
    assert not torch.equal(native, before)
    assert torch.equal(native, module)
