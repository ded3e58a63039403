"""ORACLE (test infrastructure only -- never imported by the product path).

CPU restatement of the multi-scale deformable attention operator that the reference
reaches through `mmcv` (third-party, NOT vendored in the reference tree, version
unpinned by the repo; BEVFormer's install page names mmcv-full 1.4.0):

  * `mmcv.ops.multi_scale_deform_attn.multi_scale_deformable_attn_pytorch`
      call sites: spatial_cross_attention.py:395-396, temporal_self_attention.py:252-253
  * `mmcv._ext.ms_deform_attn_forward`  (CUDA; same arithmetic, one thread per channel)
      call sites: multi_scale_deformable_attn_function.py:42-48, 118-124

Published algorithm (Deformable-DETR / mmcv): for every batch b, query q, head m

    out[b,q,m*C+c] = sum_l sum_p  w[b,q,m,l,p] * bilinear(value_l[b,:,m,c]; x*W_l-0.5, y*H_l-0.5)

with zero padding outside the map.  `msda_grid_sample` follows mmcv's CPU fallback
(per level F.grid_sample(..., bilinear, zeros, align_corners=False) on 2*loc-1);
`msda_loops` follows the CUDA kernel's scalar formulation (skip unless
-1 < h_im < H and -1 < w_im < W; corner valid iff inside) and is the bit-level
statement of the corner indexing the CUDA path must reproduce.

Parity status: UNPINNED upstream (the reference ships no tests or golden vectors,
SURVEY section 4).  Cross-checked in tests/test_oracle_cpu.py against the independent
implementation in transformers/models/mask2former/modeling_mask2former.py:798-837.
"""
import numpy as np
import torch
import torch.nn.functional as F


def msda_grid_sample(value, value_spatial_shapes, sampling_locations, attention_weights):
    """value (B, Nv, M, C); shapes (L, 2) [h, w]; loc (B, Nq, M, L, P, 2) [x, y] in [0,1];
    weights (B, Nq, M, L, P)  ->  (B, Nq, M*C)."""
    bs, _, num_heads, embed_dims = value.shape
    _, num_queries, num_heads, num_levels, num_points, _ = sampling_locations.shape
    sizes = [int(h) * int(w) for h, w in value_spatial_shapes]
    value_list = value.split(sizes, dim=1)
    grids = 2 * sampling_locations - 1
    per_level = []
    for lvl, (h, w) in enumerate(value_spatial_shapes):
        h, w = int(h), int(w)
        # (B, hw, M, C) -> (B*M, C, h, w)
        v = value_list[lvl].flatten(2).transpose(1, 2).reshape(bs * num_heads, embed_dims, h, w)
        # (B, Nq, M, P, 2) -> (B*M, Nq, P, 2)
        g = grids[:, :, :, lvl].transpose(1, 2).flatten(0, 1)
        per_level.append(F.grid_sample(v, g, mode='bilinear', padding_mode='zeros', align_corners=False))
    # (B, Nq, M, L, P) -> (B*M, 1, Nq, L*P)
    w_ = attention_weights.transpose(1, 2).reshape(bs * num_heads, 1, num_queries, num_levels * num_points)
    out = (torch.stack(per_level, dim=-2).flatten(-2) * w_).sum(-1)
    return out.view(bs, num_heads * embed_dims, num_queries).transpose(1, 2).contiguous()


def msda_loops(value, value_spatial_shapes, level_start_index, sampling_locations, attention_weights):
    """Scalar (numpy, fp32) statement of the CUDA kernel's arithmetic; small cases only."""
    v = value.detach().cpu().numpy().astype(np.float32)
    loc = sampling_locations.detach().cpu().numpy().astype(np.float32)
    aw = attention_weights.detach().cpu().numpy().astype(np.float32)
    B, Nv, M, C = v.shape
    _, Nq, _, L, P, _ = loc.shape
    out = np.zeros((B, Nq, M, C), np.float32)
    f32 = np.float32
    for b in range(B):
        for q in range(Nq):
            for m in range(M):
                acc = np.zeros(C, np.float32)
                for l in range(L):
                    H = int(value_spatial_shapes[l][0]); W = int(value_spatial_shapes[l][1])
                    base = int(level_start_index[l])
                    for p in range(P):
                        w_im = f32(loc[b, q, m, l, p, 0] * f32(W) - f32(0.5))
                        h_im = f32(loc[b, q, m, l, p, 1] * f32(H) - f32(0.5))
                        if not (h_im > -1 and w_im > -1 and h_im < H and w_im < W):
                            continue
                        h_lo = int(np.floor(h_im)); w_lo = int(np.floor(w_im))
                        lh = f32(h_im - f32(h_lo)); lw = f32(w_im - f32(w_lo))
                        hh = f32(1) - lh; hw = f32(1) - lw
                        val = np.zeros(C, np.float32)
                        if h_lo >= 0 and w_lo >= 0:
                            val += f32(hh * hw) * v[b, base + h_lo * W + w_lo, m]
                        if h_lo >= 0 and w_lo + 1 <= W - 1:
                            val += f32(hh * lw) * v[b, base + h_lo * W + w_lo + 1, m]
                        if h_lo + 1 <= H - 1 and w_lo >= 0:
                            val += f32(lh * hw) * v[b, base + (h_lo + 1) * W + w_lo, m]
                        if h_lo + 1 <= H - 1 and w_lo + 1 <= W - 1:
                            val += f32(lh * lw) * v[b, base + (h_lo + 1) * W + w_lo + 1, m]
                        acc += aw[b, q, m, l, p] * val
                out[b, q, m] = acc
    return torch.from_numpy(out.reshape(B, Nq, M * C))


U24 = 2.0 ** -24          # unit roundoff of fp32


def msda_reference(value, shapes, lsi, loc, w, grad_out=None, chunk=2048):
    """float64 restatement of mmcv's operator, forward and (with grad_out) backward, on the inputs' device.

    value (B, Nv, M, C); shapes (L, 2) [H, W]; lsi (L,) level starts in value's Nv rows (gaps allowed: only the rows a level
    addresses are read); loc (B, Nq, M, L, P, 2) [x, y]; w (B, Nq, M, L, P); grad_out (B, Nq, M*C).  mmcv's rule:
      h = y*H - 0.5, x = x*W - 0.5 (in float64 from the stored locations);
      a sample is skipped unless -1 < h < H and -1 < x < W;
      corners (floor(h) + {0, 1}, floor(x) + {0, 1}) contribute only inside the level, weights hh*hw, hh*lw, lh*hw, lh*lw;
      grad_loc = (W, H) * w * sum_c go_c * d bilinear / d(x, h), the one-sided derivative of the floor cell;
      grad_attn = sum_c go_c * bilinear_c;  grad_value scattered with index_add_.
    Where the rule differs from F.grid_sample (msda_grid_sample): at h = -1 or x = -1 exactly the sample is skipped, so
    its value and every gradient are 0, while grid_sample's autograd gives the one-sided derivative into the map.

    Returns a dict of float64 tensors:
      out (B, Nq, M*C) and out_abs = sum |w * cornerweight * v| over its terms;
      with grad_out: grad_value (B, Nv, M, C), gv_abs = sum |go * w * cornerweight| and gv_count = the number of
      (sample, corner) contributions per element (inside corners of valid samples, zero weights included: one atomic add
      each); grad_attn (B, Nq, M, L, P), ga_abs = sum_c |go_c| * sum_corners cornerweight * |v|; grad_loc
      (B, Nq, M, L, P, 2), gl_abs = (W, H) * sum_c |go_c w| * (hh(|v1|+|v2|) + lh(|v3|+|v4|), hw(|v1|+|v3|) + lw(|v2|+|v4|))
      (v1..v4 the top-left, top-right, bottom-left, bottom-right corners, 0 outside).
      Location sensitivities, for an error d in the pixel coordinates: out_dl = sum |w| (dh A_c + dx B_c), ga_dl =
      sum_c |go_c| (dh A_c + dx B_c), gv_dl = sum |go w| (dh |d cw / dh| + dx |d cw / dx|) and gl_dl = (W dh, H dx) *
      |w| sum_c |go_c| (|v1|+|v2|+|v3|+|v4|), with A_c = hw(|v1|+|v3|) + lw(|v2|+|v4|) >= |d bilinear / dh|,
      B_c = hh(|v1|+|v2|) + lh(|v3|+|v4|) >= |d bilinear / dx| and d the bound 2u(|loc * size| + 1) of fp32's rounding of
      loc * size - 0.5 (u = 2^-24).  They hold inside one pixel cell: callers keep samples away from pixel lines."""
    f64 = torch.float64
    dev = value.device
    B, Nv, M, C = value.shape
    _, Nq, _, L, P, _ = loc.shape
    shapes_h = [(int(h), int(w_)) for h, w_ in shapes.tolist()]
    starts = [int(s) for s in lsi.tolist()]
    v64 = value.to(f64)
    res = {'out': torch.zeros(B, Nq, M, C, dtype=f64, device=dev), 'out_abs': torch.zeros(B, Nq, M, C, dtype=f64, device=dev),
           'out_dl': torch.zeros(B, Nq, M, C, dtype=f64, device=dev)}
    bwd = grad_out is not None
    if bwd:
        for k in ('grad_value', 'gv_abs', 'gv_count', 'gv_dl'):
            res[k] = torch.zeros(B * Nv * M, C, dtype=f64, device=dev)
        for k in ('grad_attn', 'ga_abs', 'ga_dl'):
            res[k] = torch.zeros(B, Nq, M, L, P, dtype=f64, device=dev)
        for k in ('grad_loc', 'gl_abs', 'gl_dl'):
            res[k] = torch.zeros(B, Nq, M, L, P, 2, dtype=f64, device=dev)
        go_all = grad_out.to(f64).view(B, Nq, M, C)
    bi = torch.arange(B, device=dev).view(B, 1, 1, 1)
    mi = torch.arange(M, device=dev).view(1, 1, M, 1)
    for q0 in range(0, Nq, chunk):
        q1 = min(Nq, q0 + chunk)
        nq = q1 - q0
        if bwd:
            go = go_all[:, q0:q1, :, None, :]                                     # (B, nq, M, 1, C)
        for l, (H, W) in enumerate(shapes_h):
            xy = loc[:, q0:q1, :, l].to(f64)                                      # (B, nq, M, P, 2)
            wl = w[:, q0:q1, :, l].to(f64)                                        # (B, nq, M, P)
            x = xy[..., 0] * W - 0.5
            h = xy[..., 1] * H - 0.5
            dx = 2 * U24 * (xy[..., 0].abs() * W + 1)
            dh = 2 * U24 * (xy[..., 1].abs() * H + 1)
            valid = (h > -1) & (x > -1) & (h < H) & (x < W)
            h_lo, x_lo = torch.floor(h), torch.floor(x)
            lh, lw = h - h_lo, x - x_lo
            hh, hw = 1 - lh, 1 - lw
            h_lo, x_lo = h_lo.long(), x_lo.long()
            corners = []
            for dy, dxc in ((0, 0), (0, 1), (1, 0), (1, 1)):
                hy, wx = h_lo + dy, x_lo + dxc
                inside = valid & (hy >= 0) & (hy <= H - 1) & (wx >= 0) & (wx <= W - 1)
                pix = starts[l] + hy.clamp(0, H - 1) * W + wx.clamp(0, W - 1)       # (B, nq, M, P)
                row = (bi * Nv + pix) * M + mi                                    # row of value.view(B*Nv*M, C)
                v = v64.view(B * Nv * M, C)[row] * inside[..., None]              # (B, nq, M, P, C), 0 outside
                fy = (hh if dy == 0 else lh) * inside
                fx = (hw if dxc == 0 else lw) * inside
                corners.append((inside, row, v, fy, fx))
            (_, _, v1, _, _), (_, _, v2, _, _), (_, _, v3, _, _), (_, _, v4, _, _) = corners
            bil = sum(c[3][..., None] * c[4][..., None] * c[2] for c in corners)            # (B, nq, M, P, C)
            babs = sum(c[3][..., None] * c[4][..., None] * c[2].abs() for c in corners)
            a1, a2, a3, a4 = v1.abs(), v2.abs(), v3.abs(), v4.abs()
            A = hw[..., None] * (a1 + a3) + lw[..., None] * (a2 + a4)           # >= |d bilinear / dh|
            Bx = hh[..., None] * (a1 + a2) + lh[..., None] * (a3 + a4)           # >= |d bilinear / dx|
            sens = dh[..., None] * A + dx[..., None] * Bx
            res['out'][:, q0:q1] += (wl[..., None] * bil).sum(3)
            res['out_abs'][:, q0:q1] += (wl.abs()[..., None] * babs).sum(3)
            res['out_dl'][:, q0:q1] += (wl.abs()[..., None] * sens).sum(3)
            if not bwd:
                continue
            ago = go.abs()
            res['grad_attn'][:, q0:q1, :, l] = (go * bil).sum(-1)
            res['ga_abs'][:, q0:q1, :, l] = (ago * babs).sum(-1)
            res['ga_dl'][:, q0:q1, :, l] = (ago * sens).sum(-1)
            t = go * wl[..., None]                                                 # (B, nq, M, P, C)
            at = t.abs()
            gx = (t * (hh[..., None] * (v2 - v1) + lh[..., None] * (v4 - v3))).sum(-1)
            gy = (t * (hw[..., None] * (v3 - v1) + lw[..., None] * (v4 - v2))).sum(-1)
            res['grad_loc'][:, q0:q1, :, l, :, 0] = W * gx
            res['grad_loc'][:, q0:q1, :, l, :, 1] = H * gy
            res['gl_abs'][:, q0:q1, :, l, :, 0] = W * (at * Bx).sum(-1)
            res['gl_abs'][:, q0:q1, :, l, :, 1] = H * (at * A).sum(-1)
            dsum = (at * (a1 + a2 + a3 + a4)).sum(-1)
            res['gl_dl'][:, q0:q1, :, l, :, 0] = W * dh * dsum
            res['gl_dl'][:, q0:q1, :, l, :, 1] = H * dx * dsum
            for inside, row, _, fy, fx in corners:
                r = row[inside]
                cw = (fy * fx)[inside][:, None]
                tt = t[inside]
                res['grad_value'].index_add_(0, r, tt * cw)
                res['gv_abs'].index_add_(0, r, tt.abs() * cw)
                res['gv_count'].index_add_(0, r, torch.ones_like(tt))
                res['gv_dl'].index_add_(0, r, tt.abs() * (dh[inside][:, None] * fx[inside][:, None] +
                                                          dx[inside][:, None] * fy[inside][:, None]))
    for k in ('out', 'out_abs', 'out_dl'):
        res[k] = res[k].view(B, Nq, M * C)
    if bwd:
        for k in ('grad_value', 'gv_abs', 'gv_count', 'gv_dl'):
            res[k] = res[k].view(B, Nv, M, C)
    return res
