"""DeepCache's split of the U-Net, restated from oracle/restatement.py's helpers: `deep` runs the network up to the input
of the last up level (the feature a full pass keeps), `shallow` runs the rest from that feature -- the stem and down level
0 again for the level-0 skips, then the last up level, the final block and conv.  deep + shallow is
restatement.unet_forward; a cached pass is `shallow` on a feature another (x, t) produced.
"""
import torch
import torch.nn.functional as F

from oracle import restatement as R


def conditioning(sd, cfg, x, time, lowres_noise_times=None, text_embeds=None, text_mask=None, cond_drop_prob=0.):
    """(t, c): the time embedding and the LayerNormed conditioning tokens, as restatement.unet_forward forms them."""
    assert cond_drop_prob in (0, 0., 1, 1.)
    dim = cfg.get('dim', 128)
    bsz = x.shape[0]

    def time_branch(prefix, times):
        hid = F.silu(R._linear(sd, prefix + 'hiddens.1', R._posemb(times, dim, x.dtype)))
        return R._linear(sd, prefix + 'cond.0', hid), R._linear(sd, prefix + 'tokens.0', hid).reshape(bsz, 2, -1)
    t, tokens = time_branch('to_time_', time)
    if cfg.get('lowres_cond', False):
        lt, ltok = time_branch('to_lowres_time_', lowres_noise_times)
        t, tokens = t + lt, torch.cat((tokens, ltok), dim=-2)
    c = tokens
    if text_embeds is not None:
        max_len = sd['null_text_embed'].shape[1]
        tok = R._linear(sd, 'text_to_cond', text_embeds)[:, :max_len]
        rem = max_len - tok.shape[1]
        if rem > 0:
            tok = F.pad(tok, (0, 0, 0, rem))
        keep = torch.full((bsz,), cond_drop_prob == 0, dtype=torch.bool, device=x.device)
        keep_embed = keep[:, None, None]
        if text_mask is not None:
            tm = F.pad(text_mask, (0, rem), value=False) if rem > 0 else text_mask
            keep_embed = tm[:, :, None] & keep_embed
        tok = torch.where(keep_embed, tok, sd['null_text_embed'])
        pooled = tok.mean(dim=-2)
        p = 'to_text_non_attn_cond'
        hid = F.layer_norm(pooled, pooled.shape[-1:], sd[p + '.0.weight'], sd[p + '.0.bias'])
        hid = R._linear(sd, p + '.3', F.silu(R._linear(sd, p + '.1', hid)))
        t = t + torch.where(keep[:, None], hid, sd['null_text_hidden'])
        c = torch.cat((tokens, tok), dim=-2)
    return t, F.layer_norm(c, c.shape[-1:], sd['norm_cond.weight'], sd['norm_cond.bias'])


def _down(sd, cfg, x, i, t, c, hiddens):
    p = f'downs.{i}'
    if cfg.get('memory_efficient', False):
        x = R._conv(sd, p + '.0', x, stride=2, padding=1)
    x = R._resnet_block(sd, p + '.1', x, t, c)
    j = 0
    while f'{p}.2.{j}.block1.project.weight' in sd:
        x = R._resnet_block(sd, f'{p}.2.{j}', x, t)
        hiddens.append(x)
        j += 1
    if p + '.3.attn.fn.to_q.weight' in sd:
        x = R._transformer_block(sd, p + '.3', x, cfg.get('attn_heads', 8))
    hiddens.append(x)
    return x


def _up(sd, cfg, x, i, t, c, hiddens):
    p = f'ups.{i}'
    skip = lambda cur: torch.cat((cur, hiddens.pop() * 2 ** -0.5), dim=1)
    x = R._resnet_block(sd, p + '.0', skip(x), t, c)
    j = 0
    while f'{p}.1.{j}.block1.project.weight' in sd:
        x = R._resnet_block(sd, f'{p}.1.{j}', skip(x), t)
        j += 1
    if p + '.2.attn.fn.to_q.weight' in sd:
        x = R._transformer_block(sd, p + '.2', x, cfg.get('attn_heads', 8))
    if p + '.3.1.weight' in sd:
        x = R._conv(sd, p + '.3.1', F.interpolate(x, scale_factor=2, mode='nearest'), padding=1)
    return x


def _stem(sd, x, lowres_cond_img):
    if lowres_cond_img is not None:
        x = torch.cat((x, lowres_cond_img), dim=1)
    return torch.cat([R._conv(sd, f'init_conv.convs.{i}', x, padding=(k - 1) // 2) for i, k in enumerate((3, 7, 15))],
                     dim=1)


def deep(sd, cfg, x, time, lowres_cond_img=None, **kw):
    """The feature that enters the last up level (NCHW)."""
    L = len(tuple(cfg.get('dim_mults', (1, 2, 4))))
    t, c = conditioning(sd, cfg, x, time, **kw)
    h, hiddens = _stem(sd, x, lowres_cond_img), []
    for i in range(L):
        h = _down(sd, cfg, h, i, t, c, hiddens)
        if not cfg.get('memory_efficient', False):
            h = (R._conv(sd, f'downs.{i}.4', h, stride=2, padding=1) if i < L - 1 else
                 R._conv(sd, f'downs.{i}.4.fns.0', h, padding=1) + R._conv(sd, f'downs.{i}.4.fns.1', h))
    h = R._resnet_block(sd, 'mid_block1', h, t, c)
    if 'mid_attn.fn.fn.to_q.weight' in sd:
        tok, shp = R._tokens(h)
        h = R._untokens(R._attention(sd, 'mid_attn.fn.fn', tok, cfg.get('attn_heads', 8)), shp) + h
    h = R._resnet_block(sd, 'mid_block2', h, t, c)
    for i in range(L - 1):
        h = _up(sd, cfg, h, i, t, c, hiddens)
    return h


def shallow(sd, cfg, feature, x, time, lowres_cond_img=None, **kw):
    """The U-Net's output from `feature` (the last up level's input) and fresh level-0 skips of (x, time)."""
    L = len(tuple(cfg.get('dim_mults', (1, 2, 4))))
    t, c = conditioning(sd, cfg, x, time, **kw)
    hiddens = []
    _down(sd, cfg, _stem(sd, x, lowres_cond_img), 0, t, c, hiddens)
    h = _up(sd, cfg, feature, L - 1, t, c, hiddens)
    h = R._resnet_block(sd, 'final_res_block', h, t)
    return R._conv(sd, 'final_conv', h, padding=1)

