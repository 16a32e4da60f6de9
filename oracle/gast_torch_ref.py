"""ORACLE (test infrastructure, not product): functional PyTorch-CPU restatement of the lifting path.

Same status as oracle/gast_oracle.py (numpy): only tests/, __graft_entry__.smoke() and bench.py's
CPU-baseline / `--impl reference` leg may import it.  It exists for two reasons the numpy
restatement cannot serve:
  * it executes the SAME torch CPU kernels in the SAME order as the reference modules (conv2d,
    batch_norm, matmul on broadcast operands, cat/expand materialisations, softmax), so its
    CPU time is what the reference costs on the host cores -- this is the `cpu_baseline`;
  * it is differentiable, so it is the oracle for the training config (loss / gradients /
    running statistics) through autograd.
Pinned against the same golden vectors as the numpy oracle (tests/test_oracle_golden.py).

`p` maps state_dict keys to torch tensors; functions cite the reference file:line they follow.
"""
import torch
import torch.nn.functional as F

BN_EPS = 1e-5
BN_MOMENTUM = 0.1


def _bn(x, p, prefix, training, stats):
    """nn.BatchNorm2d(momentum=0.1) on (B,C,T,N).  In training mode uses batch statistics and
    (like the module) updates running_mean/var in place when `stats` is a dict holding them."""
    rm, rv = p[prefix + 'running_mean'], p[prefix + 'running_var']
    if training and stats is not None:
        rm = stats.setdefault(prefix + 'running_mean', rm.detach().clone())
        rv = stats.setdefault(prefix + 'running_var', rv.detach().clone())
    return F.batch_norm(x, rm if (not training or stats is not None) else None,
                        rv if (not training or stats is not None) else None,
                        p[prefix + 'weight'], p[prefix + 'bias'], training, BN_MOMENTUM, BN_EPS)


def _relu(h, tap, name):
    """F.relu, first showing its input to `tap(name, input)` when one is given (name: the BatchNorm's prefix)"""
    if tap is not None:
        tap(name, h)
    return F.relu(h)


def _dropout(h, drop, training, name):
    """F.dropout(h, drop, training) for a float `drop`; a callable `drop(name, h) -> h` instead applies a given mask
    (in training only), name being the prefix of the BatchNorm in front of this dropout"""
    if callable(drop):
        return drop(name, h) if training else h
    return F.dropout(h, drop, training)


def semch(x, W, e, mask, bias=None):
    """SemCHGraphConv.forward (model/local_attention.py:35-53)."""
    Cout = W.shape[2]
    J = mask.shape[0]
    h0 = torch.matmul(x, W[0]).unsqueeze(2).transpose(2, 4)            # :37
    h1 = torch.matmul(x, W[1]).unsqueeze(2).transpose(2, 4)            # :38
    adj = -9e15 * torch.ones(Cout, J, J, dtype=x.dtype)                # :40
    adj[mask.unsqueeze(0).expand(Cout, J, J)] = e.expand(Cout, -1).reshape(-1)   # :41
    adj = F.softmax(adj, dim=2)                                        # :42
    E = torch.eye(J, dtype=x.dtype).unsqueeze(0).repeat(Cout, 1, 1)    # :44-45
    out = torch.matmul(adj * E, h0) + torch.matmul(adj * (1 - E), h1)  # :47
    out = out.transpose(2, 4).squeeze(2)                               # :48
    return out if bias is None else out + bias.view(1, 1, -1)


def local_graph(x, p, prefix, masks, training=False, stats=None, drop=0.0, tap=None):
    """LocalGraph.forward (model/local_attention.py:130-151)."""
    sym, con = masks
    a = semch(x, p[prefix + 'gcn_sym.W'], p[prefix + 'gcn_sym.e'], sym).permute(0, 3, 1, 2)
    b = semch(x, p[prefix + 'gcn_con.W'], p[prefix + 'gcn_con.e'], con).permute(0, 3, 1, 2)
    a = _relu(_bn(a, p, prefix + 'bn_1.', training, stats), tap, prefix + 'bn_1.')
    b = _relu(_bn(b, p, prefix + 'bn_2.', training, stats), tap, prefix + 'bn_2.')
    o = torch.cat((a, b), dim=1)
    o = _relu(_bn(F.conv2d(o, p[prefix + 'cat_conv.weight']), p, prefix + 'cat_bn.', training, stats), tap,
              prefix + 'cat_bn.')
    o = _dropout(o, drop, training, prefix + 'cat_bn.')
    return o.permute(0, 2, 3, 1)


def global_graph(x, p, prefix, tap=None):
    """GlobalGraph.forward (model/global_attention.py:52-82); x: (BT, C, N)."""
    bsz = x.size(0)
    g_x = F.conv1d(x, p[prefix + 'g.weight'], p[prefix + 'g.bias']).permute(0, 2, 1)
    theta = F.conv1d(x, p[prefix + 'theta.weight'], p[prefix + 'theta.bias'])
    phi = F.conv1d(x, p[prefix + 'phi.weight'], p[prefix + 'phi.bias'])
    Ci, N = theta.shape[1], x.shape[2]
    theta_x = theta.view(bsz, Ci, -1, 1).expand(-1, -1, -1, N)
    phi_x = phi.view(bsz, Ci, 1, -1).expand(-1, -1, N, -1)
    concat = torch.cat([theta_x, phi_x], dim=1)                        # :71 (materialised)
    f = F.conv2d(concat, p[prefix + 'concat_project.0.weight']).view(bsz, N, N)   # :72
    if tap is not None:
        tap(prefix, f)                                                 # the LeakyReLU input (the logits)
    att = F.leaky_relu(f, 0.2)                                         # :74
    att = torch.add(F.softmax(att, dim=-1), p[prefix + 'C_k'])         # :76
    y = torch.matmul(att, g_x).permute(0, 2, 1).contiguous()           # :78-79
    return y


def multi_global_graph(x, p, prefix, training=False, stats=None, drop=0.0, tap=None):
    """MultiGlobalGraph.forward (model/global_attention.py:103-130)."""
    B, T, J, C = x.shape
    xf = x.contiguous().view(-1, J, C).permute(0, 2, 1)
    heads = 0
    while (prefix + 'attentions.%d.C_k' % heads) in p:
        heads += 1
    y = torch.cat([global_graph(xf, p, prefix + 'attentions.%d.' % h, tap) for h in range(heads)], dim=1)
    y = y.permute(0, 2, 1).contiguous().view(B, T, J, C).permute(0, 3, 1, 2)
    y = _relu(_bn(F.conv2d(y, p[prefix + 'cat_conv.weight']), p, prefix + 'cat_bn.', training, stats), tap,
              prefix + 'cat_bn.')
    y = _dropout(y, drop, training, prefix + 'cat_bn.')
    return y.permute(0, 2, 3, 1)


def graph_attention_block(x, p, prefix, masks, training=False, stats=None, drop=0.0, tap=None):
    """GraphAttentionBlock.forward (model/gast_net.py:22-33); x: (B,C,T,N)."""
    xl = x.permute(0, 2, 3, 1)
    a = local_graph(xl, p, prefix + 'local_graph_layer.', masks, training, stats, drop, tap)
    g = multi_global_graph(xl, p, prefix + 'global_graph_layer.', training, stats, drop, tap)
    cat = torch.cat((xl, a, g), dim=-1).permute(0, 3, 1, 2)
    return _relu(_bn(F.conv2d(cat, p[prefix + 'cat_conv.weight']), p, prefix + 'cat_bn.', training, stats), tap,
                 prefix + 'cat_bn.')


def forward(x, p, masks, filter_widths, causal=False, strided=False, dense=False,
            training=False, stats=None, drop=0.0, tap=None):
    """SpatioTemporalModel / SpatioTemporalModelOptimized1f forward (model/gast_net.py:84-104,
    159-177, 236-251).  x: (B,T,J,F) -> (B,T_out,J,3).
    `tap(name, h)`, when given, sees every kink input in forward order without changing anything: each ReLU input
    (name: the prefix of the BatchNorm in front of it) and each head's attention logits before the LeakyReLU (name:
    the head's prefix, h of shape (BT, J, J)).
    `drop` is the dropout probability, or a callable `drop(name, h)` that applies the mask of the dropout behind
    the BatchNorm `name` in training mode (tests/dropoutref.py replays the library's masks this way)."""
    fw = filter_widths
    pad = [fw[0] // 2]
    shift = [(fw[0] // 2) if causal else 0]
    nd = fw[0]
    geo = []
    for i in range(1, len(fw)):
        pad.append((fw[i] - 1) * nd // 2)
        if strided:
            shift.append((fw[i] // 2) if causal else 0)
            geo.append(dict(stride=(fw[i], 1), dilation=(1, 1)))
        else:
            shift.append((fw[i] // 2 * nd) if causal else 0)
            geo.append(dict(stride=(1, 1), dilation=(1, 1) if dense else (nd, 1)))
        nd *= fw[i]
    h = x.permute(0, 3, 1, 2)
    h = _bn(h, p, 'init_bn.', training, stats)
    h = F.conv2d(h, p['expand_conv.weight'], stride=(fw[0], 1) if strided else (1, 1))
    h = _relu(_bn(h, p, 'expand_bn.', training, stats), tap, 'expand_bn.')
    h = graph_attention_block(h, p, 'layers_graph_conv.0.', masks, training, stats, drop, tap)
    for i, g in enumerate(geo):
        if strided:
            res = h[:, :, shift[i + 1] + fw[i + 1] // 2:: fw[i + 1]]
        else:
            res = h[:, :, pad[i + 1] + shift[i + 1]: h.shape[2] - pad[i + 1] + shift[i + 1]]
        h = _relu(_bn(F.conv2d(h, p['layers_conv.%d.weight' % (2 * i)], **g), p, 'layers_bn.%d.' % (2 * i),
                      training, stats), tap, 'layers_bn.%d.' % (2 * i))
        h = _relu(_bn(F.conv2d(h, p['layers_conv.%d.weight' % (2 * i + 1)]), p, 'layers_bn.%d.' % (2 * i + 1),
                      training, stats), tap, 'layers_bn.%d.' % (2 * i + 1))
        h = res + _dropout(h, drop, training, 'layers_bn.%d.' % (2 * i + 1))
        h = graph_attention_block(h, p, 'layers_graph_conv.%d.' % (i + 1), masks, training, stats, drop, tap)
    y = F.conv2d(h, p['shrink.weight'])
    return y.permute(0, 2, 3, 1)


def mpjpe(pred, target):
    """common/loss.py:5-11."""
    assert pred.shape == target.shape
    return torch.mean(torch.norm(pred - target, dim=len(target.shape) - 1))
