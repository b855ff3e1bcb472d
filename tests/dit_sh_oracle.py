"""The DiT's Gaussian heads at gaussians_sh_degree d = 0..3, on top of oracle/dit.py (test infrastructure).

Both heads predict C = 11 + 3 (d+1)^2 channels per Gaussian, split [xyz 3 | features 3 (d+1)^2 | scaling 3 |
rotation 4 | opacity 1], and the features reshape coefficient-major, RGB-minor to [b, n, (d+1)^2, 3]
(denoiser.py:94-98, 103-120, 145-149).  Everything except the features is what oracle/dit.py computes at degree 0, so
the epilogue here hands oracle/dit.py's degree-0 epilogue the 14 channels it knows and adds the features itself; at
d = 0 every function below is the oracle/dit.py one.  Pinned to the reference's own code by
tests/test_sh_degree_cpu.py through the fixtures of tests/golden/make_dit_sh_golden.py.
"""
import torch

from oracle import dit as od


def head_channels(sh_degree):
    return 11 + 3 * (sh_degree + 1) ** 2


def _core14(t, C):
    """[.., C] raw channels -> [.., 14] = xyz | the first SH coefficient | scaling | rotation | opacity"""
    return torch.cat([t[..., :6], t[..., C - 8:]], dim=-1)


def gaussians_epilogue64(gs_tok, img_gs, ray_o, ray_d, depth_mode, sh_degree=0, near=0.0, far=500.0):
    """oracle/dit.py's gaussians_epilogue64 for gs_tok [B, G, C], img_gs [B, T, p*p*C]: features [B, P, (d+1)^2, 3]."""
    C = head_channels(sh_degree)
    b, G = gs_tok.shape[0], gs_tok.shape[1]
    img_g = img_gs.double().reshape(b, -1, C)
    pp = img_gs.shape[-1] // C
    out = od.gaussians_epilogue64(_core14(gs_tok.double(), C), _core14(img_g, C).reshape(b, -1, pp * 14), ray_o, ray_d,
                                  depth_mode, near, far)
    allg = torch.cat((gs_tok.double(), img_g), dim=1)
    out["features"] = allg[..., 3:C - 8].reshape(b, G + img_g.shape[1], (sh_degree + 1) ** 2, 3)
    return out


def heads64(model, x, mod_heads, ray_o, ray_d, depth_mode, sh_degree=0, near=0.0, far=500.0, matched=False, feed=None):
    """oracle/dit.py's heads64 at SH degree sh_degree (same arguments and outputs, gs_tok [B, G, C] and img_gs
    [B, T, p*p*C])."""
    x = x.double()
    G = model.gaussians_pos_embedding.numel() // x.shape[-1]
    D = x.shape[-1]
    mu, md = mod_heads[:, :2 * D].double(), mod_heads[:, 2 * D:].double()
    ups, dec = model.upsampler, model.image_token_decoder
    h_ups = od.modulate(od._layernorm64(x[:, :G], ups.layernorm.weight, 1e-5), mu[:, :D], mu[:, D:])
    h_dec = od.modulate(od._layernorm64(x[:, G:], dec.layernorm.weight, 1e-5), md[:, :D], md[:, D:])
    gs_tok = od._linear64(h_ups, ups.linear.weight, matched, g_bf16=False, dgrad_hi=False, wgrad_hi=False)
    img_gs = od._linear64(h_dec, dec.linear.weight, matched, g_bf16=True, dgrad_hi=True, wgrad_hi=True)
    feed = feed or {}
    fed = lambda k, v: v + (feed[k].double() - v).detach() if k in feed else v  # noqa: E731
    out = gaussians_epilogue64(fed("gs_tok", gs_tok), fed("img_gs", img_gs), ray_o, ray_d, depth_mode, sh_degree, near,
                               far)
    out.update(gs_tok=gs_tok, img_gs=img_gs, h_ups=h_ups, h_dec=h_dec)
    return out


class DenoiserOracle(od.DenoiserOracle):
    """oracle/dit.py's DenoiserOracle with heads of C = 11 + 3 (sh_degree+1)^2 channels (fp32, the reference's
    arithmetic and state_dict tree)."""

    def __init__(self, *args, sh_degree=0, **kw):
        super().__init__(*args, **kw)
        self.sh_degree = sh_degree
        C = head_channels(sh_degree)
        self.upsampler = od._Head(self.width, C)
        self.upsampler.apply(od._init_linear)
        self.image_token_decoder = od._Head(self.width, self.patch * self.patch * C)
        self.image_token_decoder.apply(od._init_linear)

    def image_to_gaussians(self, images, ray_o, ray_d, t, return_tokens=False):
        p, C = self.patch, head_channels(self.sh_degree)
        o_dot_d = torch.sum(-ray_o * ray_d, dim=2, keepdim=True)
        if self.ray_pe_type == "relative_plk":
            posed = torch.cat([images[:, :, :3] * 2.0 - 1.0, ray_d, ray_o + o_dot_d * ray_d], dim=2)
        else:
            posed = torch.cat([images[:, :, :3] * 2.0 - 1.0, torch.cross(ray_o, ray_d, dim=2), ray_d], dim=2)
        b, v, c, h, w = posed.shape
        tok = posed.reshape(b, v, c, h // p, p, w // p, p).permute(0, 1, 3, 5, 4, 6, 2).reshape(b * v, -1, p * p * c)
        tok = self.image_tokenizer(tok).reshape(b, -1, self.width)
        temb = self.t_embedder(t)
        pos = self.gaussians_pos_embedding.reshape(self.G, self.width).expand(b, -1, -1)
        x = self.transformer_input_layernorm(torch.cat((pos, tok), dim=1))
        for blk in self.transformer:
            x = blk(x, temb)
        tokens = x
        g_tok, i_tok = x.split([self.G, x.shape[1] - self.G], dim=1)
        gaussians = self.upsampler(g_tok, temb)
        img_g = self.image_token_decoder(i_tok, temb).reshape(b, -1, C)
        allg = torch.cat((gaussians, img_g), dim=1)
        xyz, features, scaling, rotation, opacity = allg.split([3, C - 11, 3, 4, 1], dim=2)
        features = features.reshape(b, -1, (self.sh_degree + 1) ** 2, 3)
        scaling = (scaling - 2.3).clamp(max=-1.20)
        opacity = opacity - 2.0
        n_img = img_g.shape[1]
        ia = xyz[:, -n_img:, :].reshape(b, v, h // p, w // p, p, p, 3).permute(0, 1, 6, 2, 4, 3, 5).reshape(b, v, 3, h, w)
        ia = ia.mean(dim=2, keepdim=True)
        if self.scene:
            depth = torch.sigmoid(ia) * (self.far - self.near) + self.near
        elif self.ray_pe_type == "relative_plk":
            depth = (2.0 * torch.sigmoid(ia) - 1.0) * 1.8 + o_dot_d
        else:
            depth = torch.sigmoid(ia)
        ia = ray_o + depth * ray_d
        ia_flat = ia.reshape(b, v, 3, h // p, p, w // p, p).permute(0, 1, 3, 5, 4, 6, 2).reshape(b, -1, 3)
        xyz = torch.cat((xyz[:, :-n_img, :], ia_flat), dim=1)
        out = dict(xyz=xyz, features=features, scaling=scaling, rotation=rotation, opacity=opacity)
        return (out, ia, tokens) if return_tokens else (out, ia)


def oracle_like(model, **kw):
    """A DenoiserOracle with the configuration of the product model `model` (DGSDenoiser[Scene]), its parameters
    loaded strictly."""
    c = model.cfg
    o = DenoiserOracle(width=c.width, heads=c.width // c.dim_heads, layers=c.num_layers, patch=c.patch_size,
                       n_gaussians=c.n_gaussians, scene=model.SCENE, near=c.range_setting_near, far=c.range_setting_far,
                       ray_pe_type=c.ray_pe_type, sh_degree=c.gaussians_sh_degree, **kw)
    o.load_state_dict({k: v.detach() for k, v in model.state_dict().items()}, strict=True)
    return o.to(model.device)
