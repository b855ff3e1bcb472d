"""Host-side logic of the batched renderer wrapper that needs no GPU: the view-chunked fallback taken when one batch
holds more than 2^31-1 instances (dgs_b200/raster.py), with the C-ABI call stubbed out."""
import torch

from dgs_b200 import raster
from dgs_b200._lib import DgsError


def test_view_chunking_on_instance_overflow_with_maps(monkeypatch):
    """The chunked fallback for plain renders and for aux=True renders, whose depth / alpha maps and their gradients are
    split across the chunks like the images."""
    calls = []

    def fake_forward(xyz, features, scaling, rotation, opacity, H, W, C2W, fxfycxcy, scale_modifier=None, arena_cache=None,
                     near_log2=None, mse_target=None, mse_loss_sum=None, aux=False):
        B, V = C2W.shape[:2]
        calls.append(V)
        if V > 2:  # "too many instances" until at most 2 views are left
            raise DgsError("libdgs_b200 status 4: instance count 2318693549 exceeds 2^31-1 (render the views in smaller batches)")
        img = C2W[:, :, 0, 3].reshape(B, V, 1, 1, 1).expand(B, V, 3, H, W).clone()  # image = the view's tag
        maps = (img[:, :, :1].clone(), 10 * img[:, :, :1]) if aux else ()  # depth = tag, alpha = 10 tag
        return (img, *maps, dict(R=100 * V, tensors=[xyz], tag=C2W[:, :, 0, 3].clone()))

    def fake_backward_one(state, grad_images, arena_cache=None, mse_coef=None, grad_depth=None, grad_alpha=None):
        # d_xyz = sum over this chunk's views of (tag * mean grad), summed over the given upstream gradients: lets the
        # test see which views each chunk got
        w = sum((state["tag"].reshape(-1) * t.mean(dim=(0, 2, 3, 4))).sum()
                for t in (grad_images, grad_depth, grad_alpha) if t is not None)
        return tuple(torch.full((1,), float(w)) for _ in range(5))

    monkeypatch.setattr(raster, "_render_batch_forward_one", fake_forward)
    real_backward = raster.render_batch_backward

    def backward(state, grad_images, arena_cache=None, mse_coef=None, grad_depth=None, grad_alpha=None):
        if "sub" in state:
            return real_backward(state, grad_images, arena_cache, mse_coef, grad_depth, grad_alpha)
        return fake_backward_one(state, grad_images, arena_cache, mse_coef, grad_depth, grad_alpha)
    monkeypatch.setattr(raster, "render_batch_backward", backward)

    B, V, H, W = 1, 7, 4, 4
    c2w = torch.zeros(B, V, 4, 4)
    c2w[0, :, 0, 3] = torch.arange(1, V + 1).float()
    fx = torch.zeros(B, V, 4)
    x = torch.zeros(B, 5, 3)
    cache = {}
    img, state = raster.render_batch_forward(x, x, x, x, x, H, W, c2w, fx, arena_cache=cache)
    # 7 -> (3, 4) -> (1, 2) and (2, 2): every view rendered exactly once, in order
    assert img.shape == (B, V, 3, H, W)
    assert torch.equal(img[0, :, 0, 0, 0], torch.arange(1, V + 1).float())
    assert state["R"] == 100 * V and raster.LAST_NUM_RENDERED == 100 * V
    assert calls == [7, 3, 1, 2, 4, 2, 2]
    g = torch.ones(B, V, 3, H, W)
    grads = raster.render_batch_backward(state, g, cache)
    assert len(grads) == 5 and float(grads[0]) == float(sum(range(1, V + 1)))
    # aux=True: the maps come back in view order, and each chunk receives its own views' map gradients
    calls.clear()
    img, depth, alpha, state = raster.render_batch_forward(x, x, x, x, x, H, W, c2w, fx, arena_cache=cache, aux=True)
    assert calls == [7, 3, 1, 2, 4, 2, 2]
    assert depth.shape == alpha.shape == (B, V, 1, H, W)
    assert torch.equal(depth[0, :, 0, 0, 0], torch.arange(1, V + 1).float()) and torch.equal(alpha, 10 * depth)
    gd = torch.ones(B, V, 1, H, W)
    grads = raster.render_batch_backward(state, None, cache, grad_depth=gd, grad_alpha=2 * gd)
    assert float(grads[0]) == 3 * float(sum(range(1, V + 1)))
    # an overflow that cannot be split any further is re-raised
    monkeypatch.setattr(raster, "_render_batch_forward_one",
                        lambda *a, **k: (_ for _ in ()).throw(DgsError("instance count 3e9 exceeds 2^31-1")))
    try:
        raster.render_batch_forward(x, x, x, x, x, H, W, c2w[:, :1], fx[:, :1])
        assert False, "expected DgsError"
    except DgsError:
        pass
