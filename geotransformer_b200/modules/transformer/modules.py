"""Transformer blocks with the reference's class names and ``state_dict`` keys; forwards run the fused sm_90a
kernels.  Reference: ``geotransformer/modules/transformer/{positional_embedding.py:8-34, rpe_transformer.py:18-131,
vanilla_transformer.py:15-129, output_layer.py:6-21, conditional_transformer.py:73-117}``.

Tensors are (N, C) (the reference carries a leading batch dimension of 1; ``GeometricTransformer`` strips and restores
it).  Masks / key weights / attention factors are ``None`` on the inference path (``EXP*/model.py:135-140``) and are
rejected explicitly if given.
"""
import numpy as np
import torch
import torch.nn as nn

from ... import functional as GF


class SinusoidalPositionalEmbedding(nn.Module):
    """reference ``positional_embedding.py:8-34``.  Only holds ``div_term``; the sinusoid itself is generated inside the
    structure-embedding kernel and never materialised."""

    def __init__(self, d_model):
        super().__init__()
        if d_model % 2 != 0:
            raise ValueError(f'Sinusoidal positional encoding with odd d_model: {d_model}')
        self.d_model = d_model
        div_indices = torch.arange(0, d_model, 2).float()
        self.register_buffer('div_term', torch.exp(div_indices * (-np.log(10000.0) / d_model)))


def _no_masks(**kw):
    for k, v in kw.items():
        if v is not None:
            raise NotImplementedError(f'{k} is not supported on the H100 inference path (always None in the reference model)')


class _WeightCache:
    """Derived, read-only copies of parameters (transposes) keyed on the parameter's version counter."""

    def __init__(self):
        self._c = {}

    def get(self, name, param, fn):
        key = (param.data_ptr(), param._version)
        hit = self._c.get(name)
        if hit is None or hit[0] != key:
            hit = (key, fn(param.detach()))
            self._c[name] = hit
        return hit[1]


class RPEMultiHeadAttention(nn.Module):
    """reference ``rpe_transformer.py:18-77``."""

    def __init__(self, d_model, num_heads, dropout=None):
        super().__init__()
        if d_model % num_heads != 0:
            raise ValueError('`d_model` ({}) must be a multiple of `num_heads` ({}).'.format(d_model, num_heads))
        if dropout:
            raise NotImplementedError('dropout is None in every shipped config')
        self.d_model, self.num_heads, self.d_model_per_head = d_model, num_heads, d_model // num_heads
        self.proj_q = nn.Linear(d_model, d_model)
        self.proj_k = nn.Linear(d_model, d_model)
        self.proj_v = nn.Linear(d_model, d_model)
        self.proj_p = nn.Linear(d_model, d_model)
        self._cache = _WeightCache()

    def forward(self, input_q, input_k, input_v, embed_qk, key_weights=None, key_masks=None, attention_factors=None):
        _no_masks(key_weights=key_weights, key_masks=key_masks, attention_factors=attention_factors)
        q = GF.linear(input_q, self.proj_q.weight, self.proj_q.bias)
        k = GF.linear(input_k, self.proj_k.weight, self.proj_k.bias)
        v = GF.linear(input_v, self.proj_v.weight, self.proj_v.bias)
        wp_t = self._cache.get('wp_t', self.proj_p.weight, lambda w: w.t().contiguous())
        qp, qb = GF.head_project(q, wp_t, self.proj_p.bias.detach(), self.num_heads)
        hidden = GF.attention(q, k, v, self.num_heads, qp=qp, qb=qb, embed=embed_qk)
        return hidden, None   # attention scores are not materialised


class MultiHeadAttention(nn.Module):
    """reference ``vanilla_transformer.py:15-75``."""

    def __init__(self, d_model, num_heads, dropout=None):
        super().__init__()
        if d_model % num_heads != 0:
            raise ValueError('`d_model` ({}) must be a multiple of `num_heads` ({}).'.format(d_model, num_heads))
        if dropout:
            raise NotImplementedError('dropout is None in every shipped config')
        self.d_model, self.num_heads, self.d_model_per_head = d_model, num_heads, d_model // num_heads
        self.proj_q = nn.Linear(d_model, d_model)
        self.proj_k = nn.Linear(d_model, d_model)
        self.proj_v = nn.Linear(d_model, d_model)

    def forward(self, input_q, input_k, input_v, key_weights=None, key_masks=None, attention_factors=None,
                attention_masks=None):
        _no_masks(key_weights=key_weights, key_masks=key_masks, attention_factors=attention_factors,
                  attention_masks=attention_masks)
        q = GF.linear(input_q, self.proj_q.weight, self.proj_q.bias)
        k = GF.linear(input_k, self.proj_k.weight, self.proj_k.bias)
        v = GF.linear(input_v, self.proj_v.weight, self.proj_v.bias)
        return GF.attention(q, k, v, self.num_heads), None


class _AttentionLayerBase(nn.Module):
    def _finish(self, hidden_states, input_states):
        hidden_states = GF.linear(hidden_states, self.linear.weight, self.linear.bias)
        return GF.add_layernorm(hidden_states, input_states, self.norm.weight, self.norm.bias, self.norm.eps)


class RPEAttentionLayer(_AttentionLayerBase):
    """reference ``rpe_transformer.py:80-107``."""

    def __init__(self, d_model, num_heads, dropout=None):
        super().__init__()
        self.attention = RPEMultiHeadAttention(d_model, num_heads, dropout=dropout)
        self.linear = nn.Linear(d_model, d_model)
        self.norm = nn.LayerNorm(d_model)

    def forward(self, input_states, memory_states, position_states, memory_weights=None, memory_masks=None,
                attention_factors=None):
        hidden, scores = self.attention(input_states, memory_states, memory_states, position_states,
                                        key_weights=memory_weights, key_masks=memory_masks,
                                        attention_factors=attention_factors)
        return self._finish(hidden, input_states), scores


class AttentionLayer(_AttentionLayerBase):
    """reference ``vanilla_transformer.py:78-105``."""

    def __init__(self, d_model, num_heads, dropout=None):
        super().__init__()
        self.attention = MultiHeadAttention(d_model, num_heads, dropout=dropout)
        self.linear = nn.Linear(d_model, d_model)
        self.norm = nn.LayerNorm(d_model)

    def forward(self, input_states, memory_states, memory_weights=None, memory_masks=None, attention_factors=None,
                attention_masks=None):
        hidden, scores = self.attention(input_states, memory_states, memory_states, key_weights=memory_weights,
                                        key_masks=memory_masks, attention_factors=attention_factors,
                                        attention_masks=attention_masks)
        return self._finish(hidden, input_states), scores


class AttentionOutput(nn.Module):
    """reference ``output_layer.py:6-21``: LN(x + squeeze(relu(expand(x))))."""

    def __init__(self, d_model, dropout=None, activation_fn='ReLU'):
        super().__init__()
        if activation_fn != 'ReLU':
            raise NotImplementedError('only ReLU (the shipped configs) is implemented')
        self.expand = nn.Linear(d_model, d_model * 2)
        self.squeeze = nn.Linear(d_model * 2, d_model)
        self.norm = nn.LayerNorm(d_model)

    def forward(self, input_states):
        h = GF.linear(input_states, self.expand.weight, self.expand.bias, relu=True)
        h = GF.linear(h, self.squeeze.weight, self.squeeze.bias)
        return GF.add_layernorm(input_states, h, self.norm.weight, self.norm.bias, self.norm.eps)


class RPETransformerLayer(nn.Module):
    """reference ``rpe_transformer.py:110-131``."""

    def __init__(self, d_model, num_heads, dropout=None, activation_fn='ReLU'):
        super().__init__()
        self.attention = RPEAttentionLayer(d_model, num_heads, dropout=dropout)
        self.output = AttentionOutput(d_model, dropout=dropout, activation_fn=activation_fn)

    def forward(self, input_states, memory_states, position_states, memory_weights=None, memory_masks=None,
                attention_factors=None):
        hidden, scores = self.attention(input_states, memory_states, position_states, memory_weights=memory_weights,
                                        memory_masks=memory_masks, attention_factors=attention_factors)
        return self.output(hidden), scores


class TransformerLayer(nn.Module):
    """reference ``vanilla_transformer.py:108-129``."""

    def __init__(self, d_model, num_heads, dropout=None, activation_fn='ReLU'):
        super().__init__()
        self.attention = AttentionLayer(d_model, num_heads, dropout=dropout)
        self.output = AttentionOutput(d_model, dropout=dropout, activation_fn=activation_fn)

    def forward(self, input_states, memory_states, memory_weights=None, memory_masks=None, attention_factors=None,
                attention_masks=None):
        hidden, scores = self.attention(input_states, memory_states, memory_weights=memory_weights,
                                        memory_masks=memory_masks, attention_factors=attention_factors,
                                        attention_masks=attention_masks)
        return self.output(hidden), scores


def _tail(layer, hidden, inp):
    """attention.linear + residual LayerNorm, then the FFN block with its residual LayerNorm (5 launches)."""
    att, ffn = layer.attention, layer.output
    h = GF.linear(hidden, att.linear.weight, att.linear.bias)
    x = GF.add_layernorm(h, inp, att.norm.weight, att.norm.bias, att.norm.eps)
    y = GF.linear(x, ffn.expand.weight, ffn.expand.bias, relu=True)
    y = GF.linear(y, ffn.squeeze.weight, ffn.squeeze.bias)
    return GF.add_layernorm(x, y, ffn.norm.weight, ffn.norm.bias, ffn.norm.eps)


def _fused(cache, mha, names, layer):
    """concatenated projection weights/biases (one GEMM instead of len(names)); cached per layer, rebuilt when ANY of the
    source parameters changes (version counters / storage)"""
    key = f'{layer}:' + '+'.join(names)
    params = [p for n in names for p in (getattr(mha, n).weight, getattr(mha, n).bias)]
    stamp = tuple((p.data_ptr(), p._version) for p in params)
    hit = cache._c.get(key)
    if hit is None or hit[0] != stamp:
        w = torch.cat([getattr(mha, n).weight.detach() for n in names], dim=0).contiguous()
        b = torch.cat([getattr(mha, n).bias.detach() for n in names], dim=0).contiguous()
        hit = (stamp, (w, b))
        cache._c[key] = hit
    return hit[1]


def _concat(mha, names):
    """the fused projection weight / bias of ``_fused``, concatenated from the parameters themselves (with their graph)"""
    return (torch.cat([getattr(mha, n).weight for n in names], dim=0), torch.cat([getattr(mha, n).bias for n in names], dim=0))


class RPEConditionalTransformer(nn.Module):
    """reference ``conditional_transformer.py:73-117`` (sequential cross updates unless ``parallel``)."""

    def __init__(self, blocks, d_model, num_heads, dropout=None, activation_fn='ReLU', return_attention_scores=False,
                 parallel=False):
        super().__init__()
        if return_attention_scores:
            raise NotImplementedError('attention scores stay on chip in the fused kernel')
        self.blocks = blocks
        layers = []
        for block in blocks:
            if block not in ('self', 'cross'):
                raise ValueError('Unsupported block type "{}".'.format(block))
            cls = RPETransformerLayer if block == 'self' else TransformerLayer
            layers.append(cls(d_model, num_heads, dropout=dropout, activation_fn=activation_fn))
        self.layers = nn.ModuleList(layers)
        self.return_attention_scores = return_attention_scores
        self.parallel = parallel
        self._cache = _WeightCache()

    def forward(self, feats0, feats1, embeddings0, embeddings1, masks0=None, masks1=None):
        _no_masks(masks0=masks0, masks1=masks1)
        n0, n1, c = feats0.shape[0], feats1.shape[0], embeddings0.shape[-1]
        E = torch.cat([embeddings0.reshape(n0 * n0, c), embeddings1.reshape(n1 * n1, c)])
        x = self.forward_stacked(torch.cat([feats0, feats1]), [n0, n1], E)
        return x[:n0], x[n0:]

    def forward_stacked(self, x, cloud_rows, embeddings):
        """The transformer over the stacked rows of B pairs, the kernel sequence of ``geob200_transformer_forward_batched``: x rows in
        stack order [ref_1..ref_B, src_1..src_B] (``cloud_rows``: their 2B row counts), ``embeddings`` the flat structure embeddings
        of the 2B clouds one after the other (sum n_c^2, C).  Every Linear / LayerNorm runs once over all rows (the ref block and the
        src block are contiguous, so a cross layer's projections are single GEMMs too); attention runs as one batched launch pair per
        phase, one item per cloud (self) or per pair (cross).  Carries the graph in grad mode when an input or a parameter requires
        grad; the kernels, and so the values, are the same either way."""
        rows = [int(r) for r in cloud_rows]
        for i in range(len(self.blocks)):
            x = self._layer(i, x, rows, embeddings)
        return x

    def _layer(self, i, x, rows, embeddings):
        """layer i of ``forward_stacked`` on the stacked rows x"""
        B, c = len(rows) // 2, x.shape[1]
        ref, src = rows[:B], rows[B:]
        layer = self.layers[i]
        mha = layer.attention.attention
        h = mha.num_heads
        if self.blocks[i] == 'self':
            (w, b), wp_t = self._weights(i, ('proj_q', 'proj_k', 'proj_v'))
            qkv = GF.linear(x, w, b)
            q, k, v = qkv[:, :c], qkv[:, c:2 * c], qkv[:, 2 * c:]
            qp, qb = GF.head_project(q, wp_t, mha.proj_p.bias, h)
            return _tail(layer, GF.attention_batched(q, k, v, h, rows, rows, qp=qp, qb=qb, embed=embeddings), x)
        (wkv, bkv), _ = self._weights(i, ('proj_k', 'proj_v'))
        R = sum(ref)
        x0, x1 = x[:R], x[R:]
        q0 = GF.linear(x0, mha.proj_q.weight, mha.proj_q.bias)
        kv1 = GF.linear(x1, wkv, bkv)
        y0 = _tail(layer, GF.attention_batched(q0, kv1[:, :c], kv1[:, c:], h, ref, src), x0)
        mem = x0 if self.parallel else y0          # the src update sees the UPDATED ref rows unless `parallel`
        q1 = GF.linear(x1, mha.proj_q.weight, mha.proj_q.bias)
        kv0 = GF.linear(mem, wkv, bkv)
        y1 = _tail(layer, GF.attention_batched(q1, kv0[:, :c], kv0[:, c:], h, src, ref), x1)
        return torch.cat([y0, y1])

    def _weights(self, i, names):
        """((w, b) of the named projections of layer i stacked for one GEMM, proj_p's transpose or None for a cross layer).  With a
        graph to the layer's parameters they are taken from the parameters themselves (autograd splits the fused gradient back onto
        each projection); without one they are the cached copies, rebuilt only when a parameter changes."""
        mha = self.layers[i].attention.attention
        rpe = isinstance(mha, RPEMultiHeadAttention)
        if GF._needs_grad(*mha.parameters()):
            return _concat(mha, names), (mha.proj_p.weight.t() if rpe else None)
        wp_t = self._cache.get(f'wp_t{i}', mha.proj_p.weight, lambda p: p.t().contiguous()) if rpe else None
        return _fused(self._cache, mha, names, i), wp_t
