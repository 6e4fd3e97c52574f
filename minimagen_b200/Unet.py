"""Denoising U-Net, H100-native (reference: minimagen/Unet.py).

Same class surface as the reference -- constructor signature (`Unet.py:31-48`), attributes (`lowres_cond`, `channels`,
`channels_out`, `text_embed_dim`, `max_text_len`, `_locals`), methods (`forward`, `forward_with_cond_scale`,
`_cast_model_parameters`, `_generate_t_tokens`, `_text_condition`), presets (`Base`, `Super`, `BaseTest`, `SuperTest`)
and an identical `state_dict()` key set, so checkpoints written by the reference load unchanged
(`generate.py:102`) -- but `forward` executes hand-written sm_90a kernels through the C ABI
(include/minimagen_b200.h): NHWC fp32 residual stream, fp16 tensor-core operands with fp32 accumulation.
"""
from typing import Union

import torch
from torch import nn

from .helpers import cast_tuple, default, exists, prob_mask_like
from .layers import (Act, Attention, Cat, Context, Conv2d, CrossEmbedLayer, Downsample, Identity, Parallel, ResnetBlock,
                     SinusoidalPosEmb, TokenView, TransformerBlock, Upsample, _no_grad_check, _ResidualAttention)
from . import _native
from .ops import get_ops
from .t5 import get_encoded_dim

F32 = torch.float32


class DeepCache:
    """Static buffers for DeepCache feature reuse (Ma et al. 2024) during sampling: the activation that enters the last up
    level (`ups[-1]`'s first ResnetBlock reads it as the current half of its skip concatenation), for `rows` batch rows.

    A store pass copies what the producer wrote -- its fp32 and/or fp16 NHWC copy, and the GroupNorm block statistics
    when its epilogue accumulated them -- into rows row0 .. row0 + b, on the device, before the consumer adds anything.  A read pass hands the consumer an Act over
    the same rows holding exactly those copies, so it takes the same route over the same bits and statistics: a read
    at the inputs of the store returns the store pass's output bit for bit.  The buffers are allocated by the first
    store (outside any graph capture: the capture's warm-up run) and kept until the cache is dropped."""

    def __init__(self, rows):
        self.rows = rows
        self.f32 = self.f16 = self.stats = None

    def store(self, act, row0):
        b = act.shape[0]
        for name in ('f32', 'f16', 'stats'):
            src = getattr(act, name)
            if src is None:
                setattr(self, name, None)
                continue
            buf = getattr(self, name)
            if buf is None or buf.shape[1:] != src.shape[1:] or buf.dtype != src.dtype:
                buf = torch.empty((self.rows, *src.shape[1:]), dtype=src.dtype, device=src.device)
                setattr(self, name, buf)
            buf[row0:row0 + b].copy_(src)

    def read(self, row0, b):
        assert self.f32 is not None or self.f16 is not None, 'a read pass needs a feature stored before it'
        rows = lambda v: None if v is None else v[row0:row0 + b]
        return Act(rows(self.f32), rows(self.f16), rows(self.stats))


class Unet(nn.Module):
    def __init__(
            self,
            *,
            dim: int = 128,
            dim_mults: tuple = (1, 2, 4),
            channels: int = 3,
            channels_out: int = None,
            cond_dim: int = None,
            text_embed_dim=get_encoded_dim('t5_small'),
            num_resnet_blocks: Union[int, tuple] = 1,
            layer_attns: Union[bool, tuple] = True,
            layer_cross_attns: Union[bool, tuple] = True,
            attn_heads: int = 8,
            lowres_cond: bool = False,
            memory_efficient: bool = False,
            attend_at_middle: bool = False
    ):
        super().__init__()
        # constructor arguments, kept for re-instantiation by `_cast_model_parameters` (reference Unet.py:81-83)
        self._locals = locals()
        self._locals.pop('self', None)
        self._locals.pop('__class__', None)

        ATTN_DIM_HEAD = 64
        NUM_TIME_TOKENS = 2
        RESNET_GROUPS = 8
        self.num_time_tokens = NUM_TIME_TOKENS

        cond_dim = default(cond_dim, dim)
        time_cond_dim = dim * 4 * (2 if lowres_cond else 1)
        self.dim, self.cond_dim, self.time_cond_dim = dim, cond_dim, time_cond_dim

        # --- time conditioning (Unet.py:101-116); index 1 of to_time_tokens is the reference's parameter-free Rearrange
        self.to_time_hiddens = nn.Sequential(SinusoidalPosEmb(dim), nn.Linear(dim, time_cond_dim), nn.SiLU())
        self.to_time_cond = nn.Sequential(nn.Linear(time_cond_dim, time_cond_dim))
        self.to_time_tokens = nn.Sequential(nn.Linear(time_cond_dim, cond_dim * NUM_TIME_TOKENS), nn.Identity())

        # --- low-res noise-level conditioning for super-resolution U-Nets (Unet.py:121-138)
        self.lowres_cond = lowres_cond
        if lowres_cond:
            self.to_lowres_time_hiddens = nn.Sequential(SinusoidalPosEmb(dim), nn.Linear(dim, time_cond_dim), nn.SiLU())
            self.to_lowres_time_cond = nn.Sequential(nn.Linear(time_cond_dim, time_cond_dim))
            self.to_lowres_time_tokens = nn.Sequential(nn.Linear(time_cond_dim, cond_dim * NUM_TIME_TOKENS),
                                                       nn.Identity())

        # --- text conditioning (Unet.py:142-161)
        self.norm_cond = nn.LayerNorm(cond_dim)
        self.text_embed_dim = text_embed_dim
        self.text_to_cond = nn.Linear(self.text_embed_dim, cond_dim)
        max_text_len = 256
        self.max_text_len = max_text_len
        self.null_text_embed = nn.Parameter(torch.randn(1, max_text_len, cond_dim))
        self.null_text_hidden = nn.Parameter(torch.randn(1, time_cond_dim))
        self.to_text_non_attn_cond = nn.Sequential(
            nn.LayerNorm(cond_dim), nn.Linear(cond_dim, time_cond_dim), nn.SiLU(),
            nn.Linear(time_cond_dim, time_cond_dim))

        # --- U-Net body (Unet.py:165-328)
        self.channels = channels
        self.channels_out = default(channels_out, channels)
        self.init_conv = CrossEmbedLayer(channels if not lowres_cond else channels * 2, dim_out=dim,
                                         kernel_sizes=(3, 7, 15), stride=1)

        dims = [dim, *map(lambda m: dim * m, dim_mults)]
        in_out = list(zip(dims[:-1], dims[1:]))
        num_resolutions = len(in_out)
        num_resnet_blocks = cast_tuple(num_resnet_blocks, num_resolutions)
        resnet_groups = cast_tuple(RESNET_GROUPS, num_resolutions)
        layer_attns = cast_tuple(layer_attns, num_resolutions)
        layer_cross_attns = cast_tuple(layer_cross_attns, num_resolutions)
        assert all(n == num_resolutions for n in map(len, (resnet_groups, layer_attns, layer_cross_attns)))

        self.skip_connect_scale = 2 ** -0.5
        self.downs = nn.ModuleList([])
        self.ups = nn.ModuleList([])
        layer_params = [num_resnet_blocks, resnet_groups, layer_attns, layer_cross_attns]
        reversed_layer_params = list(map(reversed, layer_params))

        skip_connect_dims = []
        for ind, ((dim_in, dim_out), n_blocks, groups, layer_attn, layer_cross_attn) in enumerate(
                zip(in_out, *layer_params)):
            is_last = ind == (num_resolutions - 1)
            layer_cond_dim = cond_dim if layer_cross_attn else None
            transformer_klass = TransformerBlock if layer_attn else Identity
            current_dim = dim_in
            pre_downsample = None
            if memory_efficient:
                pre_downsample = Downsample(dim_in, dim_out)
                current_dim = dim_out
            skip_connect_dims.append(current_dim)
            post_downsample = None
            if not memory_efficient:
                post_downsample = Downsample(current_dim, dim_out) if not is_last else Parallel(
                    Conv2d(dim_in, dim_out, 3, padding=1), Conv2d(dim_in, dim_out, 1))
            self.downs.append(nn.ModuleList([
                pre_downsample,
                ResnetBlock(current_dim, current_dim, cond_dim=layer_cond_dim, time_cond_dim=time_cond_dim,
                            groups=groups),
                nn.ModuleList([ResnetBlock(current_dim, current_dim, time_cond_dim=time_cond_dim, groups=groups)
                               for _ in range(n_blocks)]),
                transformer_klass(dim=current_dim, heads=attn_heads, dim_head=ATTN_DIM_HEAD),
                post_downsample,
            ]))

        mid_dim = dims[-1]
        self.mid_block1 = ResnetBlock(mid_dim, mid_dim, cond_dim=cond_dim, time_cond_dim=time_cond_dim,
                                      groups=resnet_groups[-1])
        self.mid_attn = TokenView(_ResidualAttention(
            Attention(mid_dim, heads=attn_heads, dim_head=ATTN_DIM_HEAD))) if attend_at_middle else None
        self.mid_block2 = ResnetBlock(mid_dim, mid_dim, cond_dim=cond_dim, time_cond_dim=time_cond_dim,
                                      groups=resnet_groups[-1])

        for ind, ((dim_in, dim_out), n_blocks, groups, layer_attn, layer_cross_attn) in enumerate(
                zip(reversed(in_out), *reversed_layer_params)):
            is_last = ind == (num_resolutions - 1)
            layer_cond_dim = cond_dim if layer_cross_attn else None
            transformer_klass = TransformerBlock if layer_attn else Identity
            skip_connect_dim = skip_connect_dims.pop()
            self.ups.append(nn.ModuleList([
                ResnetBlock(dim_out + skip_connect_dim, dim_out, cond_dim=layer_cond_dim,
                            time_cond_dim=time_cond_dim, groups=groups),
                nn.ModuleList([ResnetBlock(dim_out + skip_connect_dim, dim_out, time_cond_dim=time_cond_dim,
                                           groups=groups) for _ in range(n_blocks)]),
                transformer_klass(dim=dim_out, heads=attn_heads, dim_head=ATTN_DIM_HEAD),
                Upsample(dim_out, dim_in) if not is_last or memory_efficient else Identity()
            ]))

        self.init_conv_to_final_conv_residual = False
        self.final_res_block = ResnetBlock(dim, dim, time_cond_dim=time_cond_dim, groups=resnet_groups[0])
        self.final_conv = Conv2d(dim, self.channels_out, 3, padding=3 // 2)

    # -------------------------------------------------------------------------------------------- reference API
    def _cast_model_parameters(self, *, lowres_cond, text_embed_dim, channels, channels_out):
        """Return self if the settings already match, else a FRESH (randomly initialised) U-Net with the updated
        settings -- the behaviour Imagen.__init__ relies on (reference Unet.py:332-353, Imagen.py:96-101)."""
        if lowres_cond == self.lowres_cond and channels == self.channels and \
                text_embed_dim == self.text_embed_dim and channels_out == self.channels_out:
            return self
        updated = dict(lowres_cond=lowres_cond, text_embed_dim=text_embed_dim, channels=channels,
                       channels_out=channels_out)
        return self.__class__(**{**self._locals, **updated})

    def forward(self, x, time, *, lowres_cond_img=None, lowres_noise_times=None, text_embeds=None, text_mask=None,
                cond_drop_prob: float = 0.):
        """x: (b, c, s, s) fp32 NCHW noised images; time: (b,) int64.  Returns the predicted noise, (b, c_out, s, s)
        (reference signature, Unet.py:355-363)."""
        return self._forward_impl(x, time, lowres_cond_img=lowres_cond_img, lowres_noise_times=lowres_noise_times,
                                  text_embeds=text_embeds, text_mask=text_mask, cond_drop_prob=cond_drop_prob)

    def _forward_impl(self, x, *args, **kwargs):
        # kernels are enqueued on the current device's stream: make the input's device current for the duration
        with _native.device_of(x):
            if torch.is_grad_enabled() and (x.requires_grad or any(p.requires_grad for p in self.parameters())):
                # training side of the path (SURVEY 8f-2): the same network through the autograd Functions
                from .train_path import unet_forward_train
                return unet_forward_train(self, x, *args, **kwargs)
            return self._forward_dev(x, *args, **kwargs)

    def _forward_dev(self, x, time, *, lowres_cond_img=None, lowres_noise_times=None, text_embeds=None, text_mask=None,
                      cond_drop_prob: float = 0., cond_keep=None, deepcache=None):
        """x: (b, c, s, s) fp32 NCHW noised images; time: (b,) int64.  Returns the predicted noise, (b, c_out, s, s).
        Orchestration follows the reference's Unet.forward (Unet.py:355-472) block for block.
        `cond_keep` (internal, uint8/bool [b]): explicit per-sample keep mask instead of the Bernoulli(1 - cond_drop_prob)
        draw of Unet.py:587 -- lets the conditional and the unconditional pass of classifier-free guidance share one batch.
        `deepcache` (internal, sampling only): (mode, cache, row0) with a DeepCache and the first of its rows this pass
        uses.  'store' runs the whole network and keeps the feature entering ups[-1] in rows row0 .. row0 + b; 'read'
        runs only the shallowest branch on the kept feature (DeepCache docstring)."""
        assert not (self.lowres_cond and not exists(lowres_cond_img)), \
            'low resolution conditioning image must be present'
        assert not (self.lowres_cond and not exists(lowres_noise_times)), \
            'low resolution conditioning noise time must be present'
        assert deepcache is None or (deepcache[0] in ('store', 'read') and not torch.is_grad_enabled()), \
            'feature caching is for sampling: a store or read pass, under torch.no_grad()'
        B, Cx, H, W = x.shape
        device = x.device
        x = x.to(F32).contiguous()
        lowres = lowres_cond_img.to(F32).contiguous() if exists(lowres_cond_img) else None

        # conditioning for the whole batch (cheap, weight-streaming bound) on the caller's stream
        t, time_tokens = self._generate_t_tokens(time, lowres_noise_times)
        t, c = self._text_condition(text_embeds, B, cond_drop_prob, device, text_mask, t, time_tokens, cond_keep)
        # every ResnetBlock's time_mlp (SiLU -> Linear, layers.py:396-399) in ONE GEMM over the shared time embedding
        ss = self._all_scale_shifts(t)

        out = torch.empty((B, self.channels_out, H, W), dtype=F32, device=device)
        chunks = self._batch_chunks(B, x.is_cuda)
        if len(chunks) == 1:
            self._forward_body(x, lowres, t, c, ss, out, deepcache)
            return out
        # The spatial body is per-sample, so batch halves are independent: run them on two streams.  Tensor-core-bound
        # convs of one half then overlap the HBM-bound GroupNorm/cast/epilogue traffic of the other and fill each
        # other's tile-quantisation tails (fork/join is captured as parallel branches by a CUDA graph).
        main = torch.cuda.current_stream(device)
        streams = self._side_streams(len(chunks), device)
        for (b0, b1), s in zip(chunks, streams):
            s.wait_stream(main)
            with torch.cuda.stream(s):
                self._forward_body(x[b0:b1], lowres[b0:b1] if exists(lowres) else None, t[b0:b1], c[b0:b1],
                                   {k: v[b0:b1] for k, v in ss.items()}, out[b0:b1],
                                   None if deepcache is None else (deepcache[0], deepcache[1], deepcache[2] + b0))
        for s in streams:
            main.wait_stream(s)
        return out

    batch_streams = 1          # number of concurrent batch slices in forward
    min_chunk_batch = 8

    def _batch_chunks(self, B, is_cuda):
        n = self.batch_streams if is_cuda else 1
        while n > 1 and (B % n != 0 or B // n < self.min_chunk_batch):
            n -= 1
        per = B // n
        return [(i * per, (i + 1) * per) for i in range(n)]

    def _side_streams(self, n, device):
        key = (n, str(device))
        if getattr(self, "_streams_key", None) != key:
            self._streams = [torch.cuda.Stream(device=device) for _ in range(n)]
            self._streams_key = key
        return self._streams

    def _forward_body(self, x, lowres, t, c, ss, out, deepcache=None):
        """Stem -> down path -> middle -> up path -> final block/conv for a batch slice; writes NCHW into `out`."""
        from . import layers as _layers
        ops = get_ops()
        B, _, H, W = x.shape
        device = x.device
        ctx = Context(c)
        # all GroupNorm statistics accumulators of this pass come out of one zero-filled buffer (one fill, not ~180)
        n_res = sum(1 for m in self.modules() if isinstance(m, ResnetBlock))
        if x.is_cuda:
            _layers._ARENA = _layers.ZeroArena(device, B * (self.dim * max(8, 1)) // 8 * 4 * (2 * n_res + 8))
        try:
            return self._forward_body_impl(x, lowres, t, c, ss, out, ctx, deepcache)
        finally:
            _layers._ARENA = None

    def _forward_body_impl(self, x, lowres, t, c, ss, out, ctx, deepcache=None):
        ops = get_ops()
        B, _, H, W = x.shape
        device = x.device
        mode, cache, row0 = deepcache if exists(deepcache) else (None, None, 0)
        read = mode == 'read'

        # torch.cat((x, lowres_cond_img), dim=1) (Unet.py:397) + CrossEmbedLayer stem (Unet.py:400)
        h = self.init_conv.run_stem(x, lowres)

        hiddens = []
        # a read pass runs level 0 only: its skips are all the last up level pops
        for pre_downsample, init_block, resnet_blocks, attn_block, post_downsample in self.downs[:1] if read else self.downs:
            if exists(pre_downsample):
                h = pre_downsample.run(h)
            h = init_block.run(h, t, ctx, ss[init_block])
            for resnet_block in resnet_blocks:
                h = resnet_block.run(h, t, None, ss[resnet_block])
                hiddens.append(h)
            h = attn_block.run(h)
            hiddens.append(h)
            if exists(post_downsample) and not read:
                h = post_downsample.run(h)

        if not read:
            h = self.mid_block1.run(h, t, ctx, ss[self.mid_block1])
            if exists(self.mid_attn):
                h = self.mid_attn.run(h)
            h = self.mid_block2.run(h, t, ctx, ss[self.mid_block2])

        skip = lambda cur: Cat(cur, hiddens.pop(), self.skip_connect_scale)
        last = len(self.ups) - 1
        for level, (init_block, resnet_blocks, attn_block, upsample) in enumerate(self.ups):
            if read and level < last:
                continue
            if level == last and mode == 'store':
                cache.store(h, row0)
            elif level == last and read:
                h = cache.read(row0, B)
            h = init_block.run(skip(h), t, ctx, ss[init_block])
            for resnet_block in resnet_blocks:
                h = resnet_block.run(skip(h), t, None, ss[resnet_block])
            h = attn_block.run(h)
            h = upsample.run(h)

        h = self.final_res_block.run(h, t, None, ss[self.final_res_block], out_f32=False)

        # final 3x3 conv (Unet.py:472) straight into the NCHW result
        fc = self.final_conv
        if ops.igemm_supported(H, W, fc.in_channels, 16):
            fc.run_prepared_nchw(h.need_f16(), B, H, W, out)
        else:
            fc.run_prepared_nchw(h.need_f32(), B, H, W, out)

    def _all_scale_shifts(self, t):
        """{ResnetBlock: view [B, 2*dim_out] (row pitch = total width)} -- the time_mlp of every ResnetBlock evaluated
        by one fp32 GEMM  SiLU(t) @ cat(W_i)^T + cat(b_i)  (weights concatenated once and cached)."""
        from .layers import ResnetBlock
        ops = get_ops()
        blocks = [m for m in self.modules() if isinstance(m, ResnetBlock) and exists(m.time_mlp)]
        key = tuple((m.time_mlp[1].weight.data_ptr(), m.time_mlp[1].weight._version, m.time_mlp[1].bias._version)
                    for m in blocks)
        if getattr(self, "_tm_key", None) != key:
            self._tm_w = torch.cat([m.time_mlp[1].weight.detach() for m in blocks], dim=0).contiguous()
            self._tm_b = torch.cat([m.time_mlp[1].bias.detach() for m in blocks], dim=0).contiguous()
            self._tm_key = key
        B, tcd = t.shape
        total = self._tm_w.shape[0]
        st = torch.empty_like(t)
        ops.silu(t.contiguous(), st)
        buf = torch.empty((B, total), dtype=F32, device=t.device)
        ops.linear_f32(st, B, tcd, self._tm_w, self._tm_b, total, 0, 0, None, buf, None)
        out, off = {}, 0
        for m in blocks:
            n = m.time_mlp[1].out_features
            out[m] = buf[:, off:off + n]
            off += n
        return out

    def forward_with_cond_scale(self, *args, cond_scale: float = 1., **kwargs):
        """Classifier-free guidance: null + (cond - null) * cond_scale, one forward if cond_scale == 1
        (reference Unet.py:474-506)."""
        logits = self.forward(*args, **kwargs)
        if cond_scale == 1:
            return logits
        null_logits = self.forward(*args, cond_drop_prob=1., **kwargs)
        return null_logits + (logits - null_logits) * cond_scale

    def _time_branch(self, times, hiddens_seq, cond_seq, tokens_seq, t_addend):
        ops = get_ops()
        B = times.shape[0]
        dev = times.device
        tcd, D, nt = self.time_cond_dim, self.cond_dim, self.num_time_tokens
        pos = hiddens_seq[0](times)                                         # SinusoidalPosEmb -> [B, dim]
        lin = hiddens_seq[1]
        hid = torch.empty((B, tcd), dtype=F32, device=dev)
        ops.linear_f32(pos, B, lin.in_features, lin.weight, lin.bias, tcd, 0, 1, None, hid, None)   # Linear -> SiLU
        lin = cond_seq[0]
        t = torch.empty((B, tcd), dtype=F32, device=dev)
        ops.linear_f32(hid, B, tcd, lin.weight, lin.bias, tcd, 0, 0, t_addend, t, None)
        lin = tokens_seq[0]
        tok = torch.empty((B, nt * D), dtype=F32, device=dev)
        ops.linear_f32(hid, B, tcd, lin.weight, lin.bias, nt * D, 0, 0, None, tok, None)
        return t, tok.reshape(B, nt, D)

    def _generate_t_tokens(self, time, lowres_noise_times):
        """-> (t [b, time_cond_dim], time_tokens [b, 2 or 4, cond_dim])   (reference Unet.py:508-536)"""
        t, tokens = self._time_branch(time, self.to_time_hiddens, self.to_time_cond, self.to_time_tokens, None)
        if self.lowres_cond:
            t, lowres_tokens = self._time_branch(lowres_noise_times, self.to_lowres_time_hiddens,
                                                 self.to_lowres_time_cond, self.to_lowres_time_tokens, t)
            tokens = torch.cat((tokens, lowres_tokens), dim=-2)
        return t, tokens

    def _text_condition(self, text_embeds, batch_size, cond_drop_prob, device, text_mask, t, time_tokens, cond_keep=None):
        """-> (t, c): t gains the pooled-text hidden (or the learned null hidden), c = LayerNorm(cat(time tokens,
        256 text tokens with masked / dropped rows replaced by null_text_embed))   (reference Unet.py:538-634)"""
        ops = get_ops()
        B, D, tcd = batch_size, self.cond_dim, self.time_cond_dim
        nt = time_tokens.shape[1]
        has_text = exists(text_embeds)
        m = nt + (self.max_text_len if has_text else 0)
        c_pre = torch.empty((B, m, D), dtype=F32, device=device)
        ops.place_rows(time_tokens.contiguous(), B, nt, D, c_pre, m, 0)
        if has_text:
            L, E = text_embeds.shape[1], text_embeds.shape[2]
            proj = self._static_text_proj(text_embeds)           # step-invariant: projected once per sampling loop (see below)
            if proj is None:
                proj = torch.empty((B * L, D), dtype=F32, device=device)
                ops.linear_f32(text_embeds.to(F32).contiguous().reshape(B * L, E), B * L, E, self.text_to_cond.weight,
                               self.text_to_cond.bias, D, 0, 0, None, proj, None)
            keep = (cond_keep.to(device=device, dtype=torch.uint8).contiguous() if exists(cond_keep)
                    else prob_mask_like((B,), 1 - cond_drop_prob, device=device).to(torch.uint8))
            mask_u8 = text_mask.to(torch.uint8).contiguous() if exists(text_mask) else None
            pooled = torch.empty((B, D), dtype=F32, device=device)
            ops.text_tokens(proj, B, L, D, mask_u8, keep, self.null_text_embed.detach().reshape(self.max_text_len, D),
                            self.max_text_len, c_pre, m, nt, pooled)
            ln, lin1, _, lin2 = self.to_text_non_attn_cond
            pn = torch.empty((B, D), dtype=F32, device=device)
            ops.ln_rows(pooled, B, D, ln.weight, ln.bias, ln.eps, 0, None, pn, None)
            h1 = torch.empty((B, tcd), dtype=F32, device=device)
            ops.linear_f32(pn, B, D, lin1.weight, lin1.bias, tcd, 0, 1, None, h1, None)
            h2 = torch.empty((B, tcd), dtype=F32, device=device)
            ops.linear_f32(h1, B, tcd, lin2.weight, lin2.bias, tcd, 0, 0, None, h2, None)
            t_new = torch.empty((B, tcd), dtype=F32, device=device)
            ops.select_rows(h2, self.null_text_hidden.detach().reshape(tcd), keep, t, B, tcd, t_new)
            t = t_new
        c = torch.empty((B, m, D), dtype=F32, device=device)
        ops.ln_rows(c_pre.reshape(B * m, D), B * m, D, self.norm_cond.weight, self.norm_cond.bias, self.norm_cond.eps,
                    0, None, c.reshape(B * m, D), None)
        return t, c


    # ---- step-invariant conditioning (SURVEY 8a row 3 note): `text_to_cond(text_embeds)` (Unet.py:569) does not depend on the
    # timestep, yet the reference -- and a captured step graph -- recomputes it in every one of the 1000 denoising steps.  The
    # sampling loop registers its STATIC text buffer here; the projection is then computed once per loop (eagerly, outside the
    # graph) and `_text_condition` reads it.  Keyed on the buffer's address AND version, so a tensor that was modified without
    # re-registering simply misses the cache.
    def register_static_text(self, text_embeds):
        ops = get_ops()
        B, L, E = text_embeds.shape
        cache = self.__dict__.setdefault("_static_text", {})
        entry = cache.get(text_embeds.data_ptr())
        buf = entry[0] if entry is not None and entry[0].shape == (B * L, self.cond_dim) else \
            torch.empty((B * L, self.cond_dim), dtype=F32, device=text_embeds.device)
        with _native.device_of(text_embeds):
            ops.linear_f32(text_embeds.reshape(B * L, E), B * L, E, self.text_to_cond.weight, self.text_to_cond.bias,
                           self.cond_dim, 0, 0, None, buf, None)
        cache[text_embeds.data_ptr()] = (buf, text_embeds._version, self.text_to_cond.weight._version)
        return buf

    def unregister_static_text(self, text_embeds=None):
        cache = self.__dict__.get("_static_text", {})
        if text_embeds is None:
            cache.clear()
        else:
            cache.pop(text_embeds.data_ptr(), None)

    def _static_text_proj(self, text_embeds):
        entry = self.__dict__.get("_static_text", {}).get(text_embeds.data_ptr())
        if entry is None or text_embeds.dtype != F32 or not text_embeds.is_contiguous():
            return None
        buf, version, wversion = entry
        B, L, _ = text_embeds.shape
        if version != text_embeds._version or wversion != self.text_to_cond.weight._version or buf.shape[0] != B * L:
            return None
        return buf


class Base(Unet):
    """Base image-generation U-Net, original Imagen hyper-parameters (reference Unet.py:637-664)."""
    defaults = dict(
        dim=512,
        dim_mults=(1, 2, 3, 4),
        num_resnet_blocks=3,
        layer_attns=(False, True, True, True),
        layer_cross_attns=(False, True, True, True),
        memory_efficient=False
    )

    def __init__(self, *args, **kwargs):
        super().__init__(*args, **{**Base.defaults, **kwargs})


class Super(Unet):
    """Super-resolution U-Net, original Imagen hyper-parameters (reference Unet.py:667-692)."""
    defaults = dict(
        dim=128,
        dim_mults=(1, 2, 4, 8),
        num_resnet_blocks=(2, 4, 8, 8),
        layer_attns=(False, False, False, True),
        layer_cross_attns=(False, False, False, True),
        memory_efficient=True
    )

    def __init__(self, *args, **kwargs):
        super().__init__(*args, **{**Super.defaults, **kwargs})


class BaseTest(Unet):
    """Low-compute base U-Net (reference Unet.py:695-722).  NB, kept on purpose for drop-in behaviour: like the
    reference, direct construction merges `Base.defaults` (so `BaseTest()` is a dim=512 Base); the tiny config is
    obtained the way train.py does it, `Unet(**BaseTest.defaults)` via `get_default_args(BaseTest)`."""
    defaults = dict(
        dim=8,
        dim_mults=(1, 2),
        num_resnet_blocks=1,
        layer_attns=False,
        layer_cross_attns=False,
        memory_efficient=False
    )

    def __init__(self, *args, **kwargs):
        super().__init__(*args, **{**Base.defaults, **kwargs})


class SuperTest(Unet):
    """Low-compute super-resolution U-Net (reference Unet.py:725-750); same construction caveat as BaseTest."""
    defaults = dict(
        dim=8,
        dim_mults=(1, 2),
        num_resnet_blocks=(1, 2),
        layer_attns=False,
        layer_cross_attns=False,
        memory_efficient=True
    )

    def __init__(self, *args, **kwargs):
        super().__init__(*args, **{**Super.defaults, **kwargs})
