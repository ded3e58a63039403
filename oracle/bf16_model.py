"""ORACLE (test infrastructure only -- never imported by the product path).

Storage-rounding restatement of the reference's camera->occupancy hot path: the SAME algorithm as
`oracle/bevformer_occ.py` (which follows the reference file by file), with every tensor that the
bf16 / tensor-core configuration keeps in 16 bits rounded at exactly those storage points
(DESIGN.md section 3), and fp32 everywhere else.  It exists so that the parity test of the
throughput configuration can use a tight tolerance: against the fp32 oracle that configuration can
only be held to ~1e-2 (8-bit mantissas), which would hide real bugs; against this model the only
differences left are fp32 summation order, MUFU exp/log approximations (~1e-6) and the rare
round-to-nearest flips they cause.

Storage points emulated (bf16 unless noted), single frame (batch 1):
  camera tokens (feat + cams_embeds + level_embeds)            transformer_occ.py:207-227
  every nn.Linear weight (fp32 bias); BN-folded Conv3d weights
  GEMM operand copies of the BEV stream (LayerNorm outputs), bev_queries, bev_pos, prev_bev
  projected values (TSA value_proj, SCA value_proj)
  sampling offsets + attention logits: fp16
  bilinear corner weights  attention_weight * (1-dy|dy) * (1-dx|dx): bf16 (operand of the bf16xbf16->fp32 FMA)
  gather outputs (TSA after the queue mean, SCA after /count), FFN hidden, voxel features, head hidden
  the fp32 residual stream / LayerNorm / logits / flow stay fp32
  self mode (prev_bev None): sampling_offsets/attention_weights of TSA see cat([q, q+pos]); the engine
  computes it as q . (W1+W2)^T + [pos . W2^T + b] with the folded weight rounded to bf16 and the bracket a
  per-layer fp32 constant computed once from the parameters (same here)
SCA sampling location: the engine evaluates u*W + (dx - 0.5) with one rounding (fma) instead of
(u + dx/W)*W - 0.5; emulated in float64.

Parity status: this file restates the ENGINE's storage points, not the reference; its link to the
reference is that with `quant=False` (every rounding = identity) it reproduces oracle/bevformer_occ.py to fp32
round-off (<= 2e-4 on every output, tests/test_oracle_cpu.py::test_bf16_model_without_rounding_equals_fp32_oracle;
the formulation differs: direct masked SCA without the rebatch, index gather instead of grid_sample), and that
oracle is pinned bit-exactly against the unmodified reference modules (tests/golden/gen_golden.py).
"""
import torch
import torch.nn.functional as F

from . import bevformer_occ as O


class Q:
    """Rounding policy.  quant=False turns every rounding into the identity (-> the fp32 oracle's arithmetic)."""

    def __init__(self, quant=True):
        self.quant = quant

    def bf(self, x):
        return x.bfloat16().float() if self.quant else x

    def hf(self, x):
        return x.half().float() if self.quant else x


def _lin(qz, x, w, b):
    """x is already representable in its storage type; weights rounded to bf16, fp32 accumulate, fp32 bias."""
    return F.linear(x, qz.bf(w), b)


def _bilinear_gather(qz, value_t, H, W, h_im, w_im, wt):
    """value_t (M, H*W, Dh) fp32 (bf16-representable); h_im, w_im, wt (N, M, P) -> (N, M, Dh).
    mmcv kernel rules (oracle/msda.py::msda_loops): sample skipped unless -1 < h_im < H and -1 < w_im < W; a corner
    contributes iff it lies inside the map.  Corner weight = bf16(wt * (wy * wx))."""
    N, M, P = h_im.shape
    valid = (h_im > -1) & (w_im > -1) & (h_im < H) & (w_im < W)
    h_lo = torch.floor(h_im); w_lo = torch.floor(w_im)
    lh = h_im - h_lo; lw = w_im - w_lo
    hh = 1 - lh; hw = 1 - lw
    h_lo = h_lo.long(); w_lo = w_lo.long()
    out = value_t.new_zeros((N, M, value_t.shape[-1]))
    m_idx = torch.arange(M)[None, :, None].expand(N, M, P)
    for dy, dx, wy, wx in ((0, 0, hh, hw), (0, 1, hh, lw), (1, 0, lh, hw), (1, 1, lh, lw)):
        yy = h_lo + dy; xx = w_lo + dx
        inb = valid & (yy >= 0) & (yy <= H - 1) & (xx >= 0) & (xx <= W - 1)
        c = qz.bf(wt * (wy * wx)) * inb
        idx = yy.clamp(0, H - 1) * W + xx.clamp(0, W - 1)
        v = value_t[m_idx, idx]                                                  # (N, M, P, Dh)
        out += (v * c[..., None]).sum(2)
    return out


# ------------------------------------------------------------------ a5 (temporal_self_attention.py:128-272)
def tsa_gather(qz, cfg, v_prev, v_cur, qproj, bev_h, bev_w):
    """v_* (Nq, 256) projected values of queue 0 / 1; qproj (Nq, 192) = [offsets (head,queue,point,xy) | logits
    (head,queue,point)] -> (Nq, 256) = mean over the queue of MSDA (:257-262)."""
    M, P = cfg['num_heads'], cfg['tsa_points']
    Nq = bev_h * bev_w
    off = qproj[:, :M * 2 * P * 2].view(Nq, M, 2, P, 2)
    aw = qproj[:, M * 2 * P * 2:].view(Nq, M, 2, P).softmax(-1)                    # softmax over the 4 points (:209-211)
    ref = O.get_reference_points(bev_h, bev_w, dim='2d', bs=1)[0, :, 0]           # (Nq, 2) (x, y)
    out = torch.zeros(Nq, M, 32)
    for qu, v in ((0, v_prev), (1, v_cur)):
        vt = v.view(Nq, M, 32).permute(1, 0, 2).contiguous()
        w_im = (ref[:, None, None, 0] + off[:, :, qu, :, 0] / bev_w) * bev_w - 0.5       # (:224-229), x*W - 0.5
        h_im = (ref[:, None, None, 1] + off[:, :, qu, :, 1] / bev_h) * bev_h - 0.5
        out += _bilinear_gather(qz, vt, bev_h, bev_w, h_im, w_im, aw[:, :, qu])
    return qz.bf((out * 0.5).reshape(Nq, 256))


# ------------------------------------------------------------------ a6/a7 (spatial_cross_attention.py:128-175, 338-393)
def sca_gather(qz, cfg, value, qproj, ref_cam, bev_mask, level_shapes):
    """value (cams, Nv, 256) projected; qproj (Nq, 768) = [offsets (head,level,point,xy) | logits (head, level*point)];
    ref_cam (cams, Nq, D, 2), bev_mask (cams, Nq, D) -> (Nq, 256) = sum over visible cameras / max(1, #visible)."""
    M, L, P = cfg['num_heads'], cfg['num_levels'], cfg['sca_points']
    ncam, Nq, D = bev_mask.shape
    off = qproj[:, :M * L * P * 2].view(Nq, M, L, P, 2)
    aw = qproj[:, M * L * P * 2:].view(Nq, M, L * P).softmax(-1).view(Nq, M, L, P)   # over all 32 samples (:340-348)
    vis = bev_mask.sum(-1) > 0                                                      # (cams, Nq)
    slots = torch.zeros(Nq, M, 32)
    starts = [0]
    for (h, w) in level_shapes:
        starts.append(starts[-1] + h * w)
    zsel = torch.arange(P) % D                                                      # Z-anchor interleave (:366-373)
    for c in range(ncam):
        idx = vis[c].nonzero().squeeze(-1)
        if idx.numel() == 0:
            continue
        u = ref_cam[c, idx][:, zsel, 0]                                             # (n, P) anchor of point p
        v = ref_cam[c, idx][:, zsel, 1]
        acc = torch.zeros(idx.numel(), M, 32)
        for l, (H, W) in enumerate(level_shapes):
            vt = value[c, starts[l]:starts[l + 1]].view(H * W, M, 32).permute(1, 0, 2).contiguous()
            ox = off[idx, :, l, :, 0]; oy = off[idx, :, l, :, 1]                    # (n, M, P) pixel-unit offsets
            if qz.quant:                                                            # fma(u, W, dx - 0.5): one rounding
                w_im = (u[:, None, :].double() * W + (ox - 0.5).double()).float()
                h_im = (v[:, None, :].double() * H + (oy - 0.5).double()).float()
            else:                                                                   # reference order (:357-373 + op)
                w_im = (u[:, None, :] + ox / W) * W - 0.5
                h_im = (v[:, None, :] + oy / H) * H - 0.5
            acc += _bilinear_gather(qz, vt, H, W, h_im, w_im, aw[idx, :, l])
        slots[idx] += acc
    count = vis.sum(0).clamp(min=1).float()                                         # (:169-171)
    return qz.bf((slots / count[:, None, None]).reshape(Nq, 256))


def _ln(p, prefix, x):
    return F.layer_norm(x, (x.shape[-1],), p[prefix + '.weight'], p[prefix + '.bias'], 1e-5)


def encoder(qz, p, cfg, feats, img_metas, prev_bev=None):
    """-> bev (Nq, 256) fp32 = BEVFormerEncoder output for one frame.  `prev_bev` (Nq, 256) fp32, already rotated."""
    bev_h, bev_w, C = cfg['bev_h'], cfg['bev_w'], cfg['embed_dims']
    Nq = bev_h * bev_w
    pre = 'transformer'
    tokens, shapes, lsi = O.pack_camera_features(p, pre, cfg, feats)                # (cams, Nv, 1, C) fp32 adds
    tokens = qz.bf(tokens[:, :, 0])
    level_shapes = [tuple(int(v) for v in s) for s in shapes]
    pc = cfg['pc_range']
    ref_3d = O.get_reference_points(bev_h, bev_w, pc[5] - pc[2], cfg['num_points_in_pillar'], '3d', 1)
    ref_cam, bev_mask = O.point_sampling(ref_3d, pc, img_metas)
    ref_cam, bev_mask = ref_cam[:, 0], bev_mask[:, 0]
    bevq = p['bev_embedding.weight']
    pos = O.positional_encoding(p, 'positional_encoding', 1, bev_h, bev_w).flatten(2).permute(2, 0, 1)[:, 0]   # (Nq, C)
    q_f32 = bevq                                                                   # fp32 residual stream
    q_t = qz.bf(bevq)                                                              # operand copy of the current query
    q_pos_t = qz.bf(bevq + pos)
    pos_t = qz.bf(pos)
    has_prev = prev_bev is not None
    prev_t = qz.bf(prev_bev) if has_prev else None
    q0_t = q_t                                                                     # queue 1 keeps the layer-0 query (encoder.py:204-209)
    for l in range(cfg['num_layers']):
        lp = f'{pre}.encoder.layers.{l}'
        a0, a1 = lp + '.attentions.0', lp + '.attentions.1'
        d = a1 + '.deformable_attention'
        # ---- temporal self-attention
        Wv, bv = p[a0 + '.value_proj.weight'], p[a0 + '.value_proj.bias']
        v_cur = qz.bf(_lin(qz, q0_t if has_prev else q_t, Wv, bv))
        v_prev = qz.bf(_lin(qz, prev_t, Wv, bv)) if has_prev else v_cur
        Wq = torch.cat([p[a0 + '.sampling_offsets.weight'], p[a0 + '.attention_weights.weight']], 0)   # (192, 512)
        bq = torch.cat([p[a0 + '.sampling_offsets.bias'], p[a0 + '.attention_weights.bias']], 0)
        if has_prev:                                                               # cat([value[:bs] = prev_bev, q + pos])
            qp = F.linear(torch.cat([prev_t, q_pos_t], -1), qz.bf(Wq), bq)
        elif qz.quant:                                                             # folded: q . (W1+W2)^T + [pos . W2^T + b]
            qp = F.linear(q_t, qz.bf(Wq[:, :C] + Wq[:, C:])) + F.linear(pos, Wq[:, C:], bq)   # bracket: fp32 constant
        else:
            qp = F.linear(torch.cat([q_t, q_pos_t], -1), Wq, bq)
        attn = tsa_gather(qz, cfg, v_prev, v_cur, qz.hf(qp), bev_h, bev_w)
        x = _lin(qz, attn, p[a0 + '.output_proj.weight'], p[a0 + '.output_proj.bias']) + q_f32
        q_f32 = _ln(p, lp + '.norms.0', x)
        q_t = qz.bf(q_f32)
        # ---- spatial cross-attention
        Wq = torch.cat([p[d + '.sampling_offsets.weight'], p[d + '.attention_weights.weight']], 0)     # (768, 256)
        bq = torch.cat([p[d + '.sampling_offsets.bias'], p[d + '.attention_weights.bias']], 0)
        qp = qz.hf(_lin(qz, q_t, Wq, bq))
        value = qz.bf(_lin(qz, tokens, p[d + '.value_proj.weight'], p[d + '.value_proj.bias']))
        attn = sca_gather(qz, cfg, value, qp, ref_cam, bev_mask, level_shapes)
        x = _lin(qz, attn, p[a1 + '.output_proj.weight'], p[a1 + '.output_proj.bias']) + q_f32
        q_f32 = _ln(p, lp + '.norms.1', x)
        q_t = qz.bf(q_f32)
        # ---- FFN (mmcv FFN: x + W2 relu(W1 x))
        f = lp + '.ffns.0'
        h = qz.bf(F.relu(_lin(qz, q_t, p[f + '.layers.0.0.weight'], p[f + '.layers.0.0.bias'])))
        x = _lin(qz, h, p[f + '.layers.1.weight'], p[f + '.layers.1.bias']) + q_f32
        q_f32 = _ln(p, lp + '.norms.2', x)
        q_t = qz.bf(q_f32)
        q_pos_t = qz.bf(q_f32 + pos)
    return q_f32


def decoder_heads(qz, p, cfg, bev):
    """bev (Nq, 256) fp32 -> voxel features (X,Y,Z,32), occ (X,Y,Z,ncls), flow (X,Y,Z,2)."""
    bev_h, bev_w, Z = cfg['bev_h'], cfg['bev_w'], cfg['pillar_h']
    x = qz.bf(bev).t().reshape(1, -1, Z, bev_h, bev_w)                             # (1, Cmid, Z, Y, X), c = cm*Z + z
    for i in range(2):
        pre = f'transformer.decoder.{i}'
        s = p[pre + '.bn.weight'] / torch.sqrt(p[pre + '.bn.running_var'] + 1e-5)  # BN (eval) folded into the conv
        w = p[pre + '.conv.weight'] * s[:, None, None, None, None]
        b = p[pre + '.bn.bias'] - p[pre + '.bn.running_mean'] * s
        if qz.quant:
            x = qz.bf(F.relu(F.conv3d(x, qz.bf(w), b, stride=1, padding=1)))
        else:                                                                      # reference op order (conv, BN, ReLU)
            x = F.conv3d(x, p[pre + '.conv.weight'], None, stride=1, padding=1)
            x = F.batch_norm(x, p[pre + '.bn.running_mean'], p[pre + '.bn.running_var'], p[pre + '.bn.weight'],
                             p[pre + '.bn.bias'], False, 0.1, 1e-5)
            x = F.relu(x)
    vox = x.permute(0, 4, 3, 2, 1)[0]                                              # (X, Y, Z, 32)
    t = 'transformer'
    h1 = qz.bf(F.softplus(_lin(qz, vox, p[t + '.predicter.0.weight'], p[t + '.predicter.0.bias'])))
    occ = _lin(qz, h1, p[t + '.predicter.2.weight'], p[t + '.predicter.2.bias'])
    h2 = qz.bf(F.relu(_lin(qz, vox, p[t + '.flow_predicter.0.weight'], p[t + '.flow_predicter.0.bias'])))
    flow = _lin(qz, h2, p[t + '.flow_predicter.2.weight'], p[t + '.flow_predicter.2.bias'])
    return vox, occ, flow


def head_forward(p, cfg, mlvl_feats, img_metas, prev_bev=None, only_bev=False, quant=True):
    """Same contract as oracle.bevformer_occ.head_forward for batch 1: dict(bev_embed (1,C,H,W), occ, flow) (+ 'voxel').
    `prev_bev` (1, Nq, C) or (Nq, C), UN-rotated (rotated here like transformer_occ.py:189-205)."""
    qz = Q(quant)
    bev_h, bev_w = cfg['bev_h'], cfg['bev_w']
    assert mlvl_feats[0].shape[0] == 1, 'the storage-rounding model restates the single-frame engine'
    pb = None
    if prev_bev is not None:
        pb = prev_bev.reshape(bev_h * bev_w, -1).clone()
        if 'can_bus' in img_metas[0]:
            pb = O.rotate_prev_bev(pb, bev_h, bev_w, img_metas[0]['can_bus'][-1], cfg.get('rotate_center', [100, 100]))
    with torch.no_grad():
        bev = encoder(qz, p, cfg, mlvl_feats, img_metas, pb)
        if only_bev:
            return bev[None]
        vox, occ, flow = decoder_heads(qz, p, cfg, bev)
    return {'bev_embed': bev.t().reshape(1, -1, bev_h, bev_w), 'occ': occ[None], 'flow': flow[None], 'voxel': vox[None]}
