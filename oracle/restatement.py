"""TEST INFRASTRUCTURE ONLY -- CPU (torch fp32) restatement of the reference's hot path as pure functions over a
`state_dict`.  It is the oracle that travels to the GPU box (where /root/reference does not exist).

PINNING: tests/test_oracle.py checks every function here against (a) the unmodified reference imported through
oracle/reference.py (when /root/reference is present, i.e. in the build container) and (b) the committed golden
vectors tests/golden/*.pt that oracle/make_golden.py produced by running the real reference.  The reference itself has
no tests / golden vectors (SURVEY.md section 4), so those fixtures are the pin.

Only tests/, bench.py's cpu_baseline / --impl reference leg and __graft_entry__.smoke() may import this module.  The
product (minimagen_b200/) never does.

Each function cites the reference file:line it restates (paths relative to /root/reference/minimagen).
"""
import math

import torch
import torch.nn.functional as F


# ------------------------------------------------------------------------------------------------ schedule
def ddpm_tables(timesteps):
    """GaussianDiffusion.__init__ (diffusion_model.py:27-66): linear beta schedule scaled by 1000/T, everything in
    fp64, cast to fp32 at the end."""
    assert timesteps >= 20
    scale = 1000 / timesteps
    betas = torch.linspace(scale * 0.0001, scale * 0.02, timesteps, dtype=torch.float64)
    alphas = 1. - betas
    acp = torch.cumprod(alphas, 0)
    acp_prev = torch.cat((torch.ones(1, dtype=torch.float64), acp[:-1]))
    post_var = betas * (1. - acp_prev) / (1. - acp)
    tabs = dict(
        betas=betas, alphas_cumprod=acp, alphas_cumprod_prev=acp_prev,
        sqrt_alphas_cumprod=acp.sqrt(), sqrt_one_minus_alphas_cumprod=(1. - acp).sqrt(),
        log_one_minus_alphas_cumprod=(1. - acp).log(),
        sqrt_recip_alphas_cumprod=(1. / acp).sqrt(), sqrt_recipm1_alphas_cumprod=(1. / acp - 1).sqrt(),
        posterior_variance=post_var, posterior_log_variance_clipped=post_var.clamp(min=1e-20).log(),
        posterior_mean_coef1=betas * acp_prev.sqrt() / (1. - acp),
        posterior_mean_coef2=(1. - acp_prev) * alphas.sqrt() / (1. - acp))
    return {k: v.to(torch.float32) for k, v in tabs.items()}


def _ext(tab, t, x):
    """helpers.extract (helpers.py:56-67)"""
    return tab.gather(-1, t).reshape(t.shape[0], *((1,) * (x.dim() - 1)))


def q_sample(tabs, x_start, t, noise):
    """diffusion_model.py:142-147"""
    return _ext(tabs['sqrt_alphas_cumprod'], t, x_start) * x_start + \
        _ext(tabs['sqrt_one_minus_alphas_cumprod'], t, x_start) * noise


def p_sample_step(tabs, x, t, eps, noise, percentile=0.9):
    """Imagen._p_mean_variance + _p_sample after the U-Net (Imagen.py:307-326, :361-370):
    x0 prediction, dynamic threshold via torch.quantile, clamp/divide, posterior mean, noise add."""
    x0 = _ext(tabs['sqrt_recip_alphas_cumprod'], t, x) * x - _ext(tabs['sqrt_recipm1_alphas_cumprod'], t, x) * eps
    s = torch.quantile(x0.flatten(1).abs(), percentile, dim=-1)
    s.clamp_(min=1.)
    s = s.reshape(-1, *((1,) * (x.dim() - 1)))
    x0 = x0.clamp(-s, s) / s
    mean = _ext(tabs['posterior_mean_coef1'], t, x) * x0 + _ext(tabs['posterior_mean_coef2'], t, x) * x
    log_var = _ext(tabs['posterior_log_variance_clipped'], t, x)
    nonzero = (1 - (t == 0).float()).reshape(x.shape[0], *((1,) * (x.dim() - 1)))
    return mean + nonzero * (0.5 * log_var).exp() * noise


def cfg_combine(eps_cond, eps_null, cond_scale):
    """Unet.forward_with_cond_scale (Unet.py:506)"""
    return eps_null + (eps_cond - eps_null) * cond_scale


# ------------------------------------------------------------------------------------------------ layers
def _conv(sd, p, x, stride=1, padding=0):
    return F.conv2d(x, sd[p + '.weight'], sd.get(p + '.bias'), stride=stride, padding=padding)


def _linear(sd, p, x):
    return F.linear(x, sd[p + '.weight'], sd.get(p + '.bias'))


def _ln(sd, p, x):
    """layers.LayerNorm (layers.py:333-343): gamma parameter + zero beta buffer"""
    return F.layer_norm(x, x.shape[-1:], sd[p + '.gamma'], sd[p + '.beta'])


def _chan_ln(sd, p, x, eps=1e-5):
    """layers.ChanLayerNorm (layers.py:164-177)"""
    var = x.var(dim=1, unbiased=False, keepdim=True)
    mean = x.mean(dim=1, keepdim=True)
    return (x - mean) / (var + eps).sqrt() * sd[p + '.g']


def _posemb(t, dim, dtype=torch.float32):
    """layers.SinusoidalPosEmb (layers.py:455-465); `dtype` float64 for a float64 run of the network"""
    half = dim // 2
    step = math.log(10000) / (half - 1)
    ar = torch.arange(half, device=t.device)
    freqs = torch.exp((ar.double() if dtype == torch.float64 else ar) * -step)
    arg = t[:, None] * freqs[None, :]
    return torch.cat((arg.sin(), arg.cos()), dim=-1)


def _block(sd, p, x, scale_shift=None, groups=8):
    """layers.Block.forward (layers.py:131-145)"""
    x = F.group_norm(x, groups, sd[p + '.groupnorm.weight'], sd[p + '.groupnorm.bias'], 1e-5)
    if scale_shift is not None:
        scale, shift = scale_shift
        x = x * (scale + 1) + shift
    return _conv(sd, p + '.project', F.silu(x), padding=1)


def _softmax_dtype(sim):
    """The reference softmaxes in fp32 whatever it is fed; a float64 run of this restatement stays float64."""
    return torch.float64 if sim.dtype == torch.float64 else torch.float32


def _split_heads(x, h):
    b, n, _ = x.shape
    return x.reshape(b, n, h, -1).permute(0, 2, 1, 3)


def _cross_attention(sd, p, x, context, heads=8, mask=None):
    """layers.CrossAttention.forward (layers.py:220-251); x [b, n, c], context [b, m, d] (not normed)"""
    b = x.shape[0]
    xn = _ln(sd, p + '.norm', x)
    q = F.linear(xn, sd[p + '.to_q.weight'])
    k, v = F.linear(context, sd[p + '.to_kv.weight']).chunk(2, dim=-1)
    q, k, v = (_split_heads(t, heads) for t in (q, k, v))
    nk, nv = sd[p + '.null_kv'].unbind(dim=0)
    k = torch.cat((nk.expand(b, heads, 1, -1), k), dim=-2)
    v = torch.cat((nv.expand(b, heads, 1, -1), v), dim=-2)
    q = q * (q.shape[-1] ** -0.5)
    sim = q @ k.transpose(-1, -2)
    if mask is not None:
        mk = F.pad(mask, (1, 0), value=True)[:, None, None, :]
        sim = sim.masked_fill(~mk, -torch.finfo(sim.dtype).max)
    out = sim.softmax(dim=-1, dtype=_softmax_dtype(sim)) @ v
    out = out.permute(0, 2, 1, 3).reshape(b, x.shape[1], -1)
    return _ln(sd, p + '.to_out.1', F.linear(out, sd[p + '.to_out.0.weight']))


def _attention(sd, p, x, heads=8, mask=None):
    """layers.Attention.forward (layers.py:52-104): multi-query -- one shared k/v head"""
    b = x.shape[0]
    xn = _ln(sd, p + '.norm', x)
    q = _split_heads(F.linear(xn, sd[p + '.to_q.weight']), heads)
    k, v = F.linear(xn, sd[p + '.to_kv.weight']).chunk(2, dim=-1)           # [b, n, 64] each
    q = q * (q.shape[-1] ** -0.5)
    nk, nv = sd[p + '.null_kv'].unbind(dim=0)
    k = torch.cat((nk.expand(b, 1, -1), k), dim=-2)
    v = torch.cat((nv.expand(b, 1, -1), v), dim=-2)
    sim = torch.einsum('bhid,bjd->bhij', q, k)
    if mask is not None:
        mk = F.pad(mask, (1, 0), value=True)[:, None, None, :]
        sim = sim.masked_fill(~mk, -torch.finfo(sim.dtype).max)
    out = torch.einsum('bhij,bjd->bhid', sim.softmax(dim=-1, dtype=_softmax_dtype(sim)), v)
    out = out.permute(0, 2, 1, 3).reshape(b, x.shape[1], -1)
    return _ln(sd, p + '.to_out.1', F.linear(out, sd[p + '.to_out.0.weight']))


def _tokens(x):
    b, c, h, w = x.shape
    return x.flatten(2).transpose(1, 2), (b, c, h, w)


def _untokens(t, shp):
    b, c, h, w = shp
    return t.transpose(1, 2).reshape(b, c, h, w)


def _resnet_block(sd, p, x, t=None, c=None):
    """layers.ResnetBlock.forward (layers.py:417-439)"""
    scale_shift = None
    if (p + '.time_mlp.1.weight') in sd and t is not None:
        te = _linear(sd, p + '.time_mlp.1', F.silu(t))[:, :, None, None]
        scale_shift = te.chunk(2, dim=1)
    h = _block(sd, p + '.block1', x)
    if (p + '.cross_attn.fn.to_q.weight') in sd:
        tok, shp = _tokens(h)
        h = _untokens(_cross_attention(sd, p + '.cross_attn.fn', tok, c), shp) + h
    h = _block(sd, p + '.block2', h, scale_shift)
    res = _conv(sd, p + '.res_conv', x) if (p + '.res_conv.weight') in sd else x
    return h + res


def _transformer_block(sd, p, x, heads=8):
    """layers.TransformerBlock.forward (layers.py:496-499) + ChanFeedForward (layers.py:148-161)"""
    tok, shp = _tokens(x)
    x = _untokens(_attention(sd, p + '.attn.fn', tok, heads), shp) + x
    h = _conv(sd, p + '.ff.1', _chan_ln(sd, p + '.ff.0', x))
    h = _conv(sd, p + '.ff.4', _chan_ln(sd, p + '.ff.3', F.gelu(h)))
    return h + x


# ------------------------------------------------------------------------------------------------ U-Net
def unet_forward(sd, cfg, x, time, lowres_cond_img=None, lowres_noise_times=None, text_embeds=None, text_mask=None,
                 cond_drop_prob=0.):
    """Unet.forward (Unet.py:355-472) incl. _generate_t_tokens (:508-536) and _text_condition (:538-634).
    cfg: the Unet constructor kwargs (dim, dim_mults, num_resnet_blocks, layer_attns, lowres_cond, memory_efficient,
    attend_at_middle, attn_heads).  cond_drop_prob must be 0 or 1 (sampling), so no RNG is involved."""
    assert cond_drop_prob in (0, 0., 1, 1.)
    dim = cfg.get('dim', 128)
    mults = tuple(cfg.get('dim_mults', (1, 2, 4)))
    L = len(mults)
    heads = cfg.get('attn_heads', 8)
    lowres = cfg.get('lowres_cond', False)
    mem_eff = cfg.get('memory_efficient', False)
    bsz = x.shape[0]

    # --- time conditioning
    def time_branch(prefix, times):
        hid = F.silu(_linear(sd, prefix + 'hiddens.1', _posemb(times, dim, x.dtype)))
        return _linear(sd, prefix + 'cond.0', hid), _linear(sd, prefix + 'tokens.0', hid).reshape(bsz, 2, -1)
    t, time_tokens = time_branch('to_time_', time)
    if lowres:
        lt, ltok = time_branch('to_lowres_time_', lowres_noise_times)
        t = t + lt
        time_tokens = torch.cat((time_tokens, ltok), dim=-2)

    # --- text conditioning
    text_tokens = None
    if text_embeds is not None:
        max_len = sd['null_text_embed'].shape[1]
        tok = _linear(sd, 'text_to_cond', text_embeds)[:, :max_len]
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
        hid = _linear(sd, p + '.3', F.silu(_linear(sd, p + '.1', hid)))
        hid = torch.where(keep[:, None], hid, sd['null_text_hidden'])
        t = t + hid
        text_tokens = tok
    c = time_tokens if text_tokens is None else torch.cat((time_tokens, text_tokens), dim=-2)
    c = F.layer_norm(c, c.shape[-1:], sd['norm_cond.weight'], sd['norm_cond.bias'])

    # --- body
    if lowres_cond_img is not None:
        x = torch.cat((x, lowres_cond_img), dim=1)
    x = torch.cat([_conv(sd, f'init_conv.convs.{i}', x, padding=(k - 1) // 2) for i, k in enumerate((3, 7, 15))], dim=1)

    hiddens = []
    for i in range(L):
        p = f'downs.{i}'
        if mem_eff:
            x = _conv(sd, p + '.0', x, stride=2, padding=1)
        x = _resnet_block(sd, p + '.1', x, t, c)
        j = 0
        while (f'{p}.2.{j}.block1.project.weight') in sd:
            x = _resnet_block(sd, f'{p}.2.{j}', x, t)
            hiddens.append(x)
            j += 1
        if (p + '.3.attn.fn.to_q.weight') in sd:
            x = _transformer_block(sd, p + '.3', x, heads)
        hiddens.append(x)
        if not mem_eff:
            if i < L - 1:
                x = _conv(sd, p + '.4', x, stride=2, padding=1)
            else:
                x = _conv(sd, p + '.4.fns.0', x, padding=1) + _conv(sd, p + '.4.fns.1', x)

    x = _resnet_block(sd, 'mid_block1', x, t, c)
    if 'mid_attn.fn.fn.to_q.weight' in sd:
        tok, shp = _tokens(x)
        x = _untokens(_attention(sd, 'mid_attn.fn.fn', tok, heads), shp) + x
    x = _resnet_block(sd, 'mid_block2', x, t, c)

    skip = lambda cur: torch.cat((cur, hiddens.pop() * 2 ** -0.5), dim=1)
    for i in range(L):
        p = f'ups.{i}'
        x = _resnet_block(sd, p + '.0', skip(x), t, c)
        j = 0
        while (f'{p}.1.{j}.block1.project.weight') in sd:
            x = _resnet_block(sd, f'{p}.1.{j}', skip(x), t)
            j += 1
        if (p + '.2.attn.fn.to_q.weight') in sd:
            x = _transformer_block(sd, p + '.2', x, heads)
        if (p + '.3.1.weight') in sd:
            x = _conv(sd, p + '.3.1', F.interpolate(x, scale_factor=2, mode='nearest'), padding=1)

    x = _resnet_block(sd, 'final_res_block', x, t)
    return _conv(sd, 'final_conv', x, padding=1)
