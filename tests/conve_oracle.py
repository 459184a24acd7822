"""Float64 restatement of the ConvE decoder (DESIGN.md section 1), the yardstick of the ConvE tests."""
import torch
import torch.nn.functional as Fn


def query_rows(codes, rel, rel_inv, filters, conv_bias, W_fc, b_fc, h, anchors, relations, sides, masks=None,
               keeps=(1.0, 1.0, 1.0)):
    """q [n, d] of the queries (anchor, relation, side): image [codes[a] ; rel[r] or rel_inv[r]] as 2h x w, input
    dropout, 3x3 filters + bias, ReLU, feature dropout, W_fc + b_fc, hidden dropout, ReLU.  masks: (input [n, 2d],
    feature [n, C], hidden [n, d]) keep-masks or None each."""
    n, d = len(anchors), codes.shape[1]
    w = d // h
    sides = torch.as_tensor(sides, device=codes.device).bool()
    rho = torch.where(sides[:, None], rel[relations], rel_inv[relations])
    img = torch.cat([codes[anchors], rho], 1)
    m_in, m_feat, m_hid = masks if masks is not None else (None, None, None)
    if m_in is not None:
        img = img * m_in.to(img.dtype) / keeps[0]
    x = Fn.conv2d(img.reshape(n, 1, 2 * h, w), filters[:, None], conv_bias)
    x = torch.relu(x)
    if m_feat is not None:
        x = x * m_feat.to(x.dtype)[:, :, None, None] / keeps[1]
    z = x.reshape(n, -1) @ W_fc + b_fc
    if m_hid is not None:
        z = z * m_hid.to(z.dtype) / keeps[2]
    return torch.relu(z)


def one_to_n_loss(codes, rel, rel_inv, filters, conv_bias, W_fc, b_fc, h, queries, labels, smoothing, masks=None,
                  keeps=(1.0, 1.0, 1.0)):
    """(loss, reg): the mean over n V of the sigmoid cross-entropy of q . codes[v] against y' = (1 - eps) y + eps / V
    (labels a bool [n, V]), and (|codes[a]|^2 + |rho|^2) / (n d) summed over the queries."""
    q = torch.as_tensor(queries, device=codes.device).long()
    a, r, s = q[:, 0], q[:, 1], q[:, 2]
    Q = query_rows(codes, rel, rel_inv, filters, conv_bias, W_fc, b_fc, h, a, r, s, masks, keeps)
    E = Q @ codes.T
    n, V = E.shape
    y = labels.to(E.dtype) * (1.0 - smoothing) + smoothing / V
    loss = Fn.binary_cross_entropy_with_logits(E, y, reduction='sum') / (n * V)
    rho = torch.where(s.bool()[:, None], rel[r], rel_inv[r])
    reg = ((codes[a] ** 2).sum() + (rho ** 2).sum()) / (n * codes.shape[1])
    return loss, reg


def ranks(scores, gold, known=None):
    """raw = #{v : score_v >= gold score} (the gold always counts), filtered = raw - #{known v counted} + 1."""
    g = scores.gather(1, gold[:, None])
    ge = scores >= g
    ge[torch.arange(len(gold)), gold] = True
    raw = ge.sum(1)
    filt = None if known is None else raw - (ge & known).sum(1) + 1
    return raw, filt
