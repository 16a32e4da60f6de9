"""The training forward's dropout masks in numpy, bit for bit.

The library draws every mask with a counter-based hash (csrc/train_kernels.cuh: dropout_mask_kernel): element i of the
k-th dropout site of a forward (1-based, in forward order) is kept when

    s = seed + 0x51ED270B * k + dstate                      (mod 2^64)
    x = i * 0x9E3779B97F4A7C15 + s, then the splitmix64 finaliser
    u = float32(x >> 40) * 2^-24 >= float32(p)

and a kept value is multiplied by float32(1) / (float32(1) - float32(p)).  `seed` is the one value the engine draws
per training forward, `torch.randint(0, 2**62, (1,))` on torch's CPU generator, so `torch.manual_seed` fixes it;
`dstate` is the device-side counter a graph-capturing trainer adds (0 otherwise), advanced by DSTATE_STEP per forward.
With the masks restated here they can be injected into the fp64 port (oracle/gast_torch_ref.py, `drop=` a callable)
and into the unmodified reference, and every gradient under dropout held to the same bars as at dropout 0.

Sites, in forward order for L stages: per stage s, the residual tail `layers_bn.{2s-1}.` (s >= 1 only), then the
LocalGraph tail `layers_graph_conv.{s}.local_graph_layer.cat_bn.`, then the MultiGlobalGraph tail
`layers_graph_conv.{s}.global_graph_layer.cat_bn.`: 3L - 1 sites, each named by the BatchNorm in front of it.  A site's
mask covers its whole output (training computes every position) in row-major (b, t, j, c) order.
"""
import numpy as np
import torch

SITE_MUL = 0x51ED270B
GOLDEN_GAMMA = 0x9E3779B97F4A7C15
MIX1 = 0xBF58476D1CE4E5B9
MIX2 = 0x94D049BB133111EB
DSTATE_STEP = 0xD1B54A32D192ED03       # dropout_bump_kernel: the device counter's advance per forward
U64 = (1 << 64) - 1


def site_seed(seed, k, dstate=0):
    """the hash offset of site k (1-based) for the forward seed `seed` and device counter `dstate`"""
    return (int(seed) + SITE_MUL * int(k) + int(dstate)) & U64


def bits(seed, k, idx, dstate=0):
    """the mixed 64-bit hash x of the elements `idx` (uint64 array) of site k"""
    s = np.uint64(site_seed(seed, k, dstate))
    with np.errstate(over='ignore'):
        x = np.asarray(idx, dtype=np.uint64) * np.uint64(GOLDEN_GAMMA) + s
        x ^= x >> np.uint64(30)
        x *= np.uint64(MIX1)
        x ^= x >> np.uint64(27)
        x *= np.uint64(MIX2)
        x ^= x >> np.uint64(31)
    return x


def uniform(x):
    """u = float32(x >> 40) * 2^-24 (exact: x >> 40 has 24 bits)"""
    return (x >> np.uint64(40)).astype(np.float32) * np.float32(2.0 ** -24)


def keep(seed, k, n, p, dstate=0):
    """the uint8 keep mask of the n elements of site k"""
    return (uniform(bits(seed, k, np.arange(n, dtype=np.uint64), dstate)) >= np.float32(p)).astype(np.uint8)


def scale(p):
    """the device's factor of a kept value (F.dropout's 1 / (1 - p) can differ in the last bits)"""
    return np.float32(1) / (np.float32(1) - np.float32(p))


def engine_seed(S):
    """the seed the engine draws in a training forward that directly follows torch.manual_seed(S)"""
    g = torch.Generator().manual_seed(int(S))
    return int(torch.randint(0, 2 ** 62, (1,), generator=g).item())


def dstate_value(t):
    """the device counter (an int64 tensor of one element, as GraphedTrainer keeps it) as the unsigned value added"""
    return int(t.item()) & U64


def sites(L):
    """the dropout sites of an L-stage model in forward order, by the prefix of the BatchNorm in front of each"""
    out = []
    for s in range(L):
        if s >= 1:
            out.append('layers_bn.%d.' % (2 * s - 1))
        out.append('layers_graph_conv.%d.local_graph_layer.cat_bn.' % s)
        out.append('layers_graph_conv.%d.global_graph_layer.cat_bn.' % s)
    return out


def _arch(case_or_arch):
    """(filter widths, channels, strided) of a kinkfree.Case or of a golden's meta dict"""
    if isinstance(case_or_arch, dict):
        m = case_or_arch
        return list(m['filter_widths']), m['channels'], m['strided']
    c = case_or_arch
    return list(c.fw), c.ch, c.strided


def stage_frames(fw, T, strided):
    """the frames of every stage's output in a training forward over T input frames (the dense ablation's kernels
    span what the dilated ones do)"""
    t = (T - fw[0]) // fw[0] + 1 if strided else T - fw[0] + 1
    out, nd = [t], fw[0]
    for w in fw[1:]:
        t = (t - w) // w + 1 if strided else t - (w - 1) * nd
        out.append(t)
        nd *= w
    return out


def site_shapes(case_or_arch, B, T, J):
    """{site: (B, C, T_l, J)}, the shape of the port's (and the reference's) tensor at every site"""
    fw, ch, strided = _arch(case_or_arch)
    frames = stage_frames(fw, T, strided)
    names = sites(len(fw))
    shapes = {}
    for name in names:
        s = int(name.split('.')[1])
        s = (s + 1) // 2 if name.startswith('layers_bn.') else s
        shapes[name] = (B, ch << s, frames[s], J)
    return shapes


def to_port(flat, shape, p):
    """a site's keep mask in (b, t, j, c) order -> the scaled fp64 mask of the port's (B, C, T, J) tensor"""
    B, C, T, J = shape
    m = torch.from_numpy(np.ascontiguousarray(flat).reshape(B, T, J, C)).permute(0, 3, 1, 2).double()
    return m * float(scale(p))


def masks(case_or_arch, B, T, J, p, seed, dstate=0):
    """{site prefix: the scaled fp64 mask tensor (B, C, T_l, J)} of one training forward"""
    shapes = site_shapes(case_or_arch, B, T, J)
    return {name: to_port(keep(seed, k + 1, int(np.prod(shapes[name])), p, dstate), shapes[name], p)
            for k, name in enumerate(sites(len(_arch(case_or_arch)[0])))}


def dropper(mask_dict):
    """`drop(name, h)` for oracle/gast_torch_ref.py: h times the site's scaled mask"""
    def drop(name, h):
        m = mask_dict[name]
        assert tuple(m.shape) == tuple(h.shape), (name, tuple(m.shape), tuple(h.shape))
        return h * m.to(h.dtype)
    return drop


def pack(mask_dict):
    """{site: packed keep bits in (b, t, j, c) order} for a golden file"""
    return {name: np.packbits((m.permute(0, 2, 3, 1).reshape(-1) != 0).numpy().astype(np.uint8))
            for name, m in mask_dict.items()}


def unpack(packed, shape, p):
    """a site's packed keep bits (pack) -> its scaled fp64 mask"""
    return to_port(np.unpackbits(packed)[:int(np.prod(shape))], shape, p)


def golden_masks(g):
    """the masks a golden with `drop_seed` in its meta was made with, from the packed bits it stores"""
    meta = g['meta']
    shapes = site_shapes(meta, meta['B'], meta['T'], meta['J'])
    return {name: unpack(g['keep/' + name], shapes[name], meta['dropout']) for name in sites(len(meta['filter_widths']))}
