"""Shared generators and comparison helpers for the parity tests (SURVEY.md section 8d inputs)."""
import numpy as np


def random_boxes(n, seed, width=1000, height=600, smin=16, smax=512, integer=False):
    """centres uniform, sizes log-uniform [smin, smax], clipped to the image."""
    rng = np.random.default_rng(seed)
    cx = rng.uniform(0, width, n)
    cy = rng.uniform(0, height, n)
    w = np.exp(rng.uniform(np.log(smin), np.log(smax), n))
    h = np.exp(rng.uniform(np.log(smin), np.log(smax), n))
    b = np.stack([cx - w / 2, cy - h / 2, cx + w / 2, cy + h / 2], axis=1)
    b[:, 0::2] = np.clip(b[:, 0::2], 0, width - 1)
    b[:, 1::2] = np.clip(b[:, 1::2], 0, height - 1)
    if integer:
        b = np.round(b)
    return b.astype(np.float32)


def tie_free_scores(n, seed, lo=0.001, hi=0.999):
    rng = np.random.default_rng(seed)
    return rng.permutation(np.linspace(lo, hi, n)).astype(np.float32)


def iou_matrix64(b):
    """float64 IoU (+1 convention) of every pair, for margin checks."""
    b = b.astype(np.float64)
    area = (b[:, 2] - b[:, 0] + 1) * (b[:, 3] - b[:, 1] + 1)
    iw = np.minimum(b[:, None, 2], b[None, :, 2]) - np.maximum(b[:, None, 0], b[None, :, 0]) + 1
    ih = np.minimum(b[:, None, 3], b[None, :, 3]) - np.maximum(b[:, None, 1], b[None, :, 1]) + 1
    inter = np.clip(iw, 0, None) * np.clip(ih, 0, None)
    return inter / (area[:, None] + area[None, :] - inter)


def nudge_off_threshold(boxes, thresh, margin=1e-5, max_rounds=20, seed=0):
    """Perturb boxes until no pair's IoU lies within `margin` of `thresh`, so that fp32 rounding /
    FMA-contraction differences between implementations cannot flip a comparison."""
    rng = np.random.default_rng(seed)
    b = boxes.copy()
    for _ in range(max_rounds):
        iou = iou_matrix64(b)
        np.fill_diagonal(iou, 0)
        bad = np.where(np.abs(iou - thresh) < margin)
        if bad[0].size == 0:
            return b
        idx = np.unique(bad[0])
        b[idx, 2] += rng.uniform(0.25, 0.75, idx.size).astype(np.float32)
    raise AssertionError("could not separate IoUs from threshold")


def rel_err(a, b):
    a = np.asarray(a, dtype=np.float64)
    b = np.asarray(b, dtype=np.float64)
    denom = max(np.abs(b).max(), 1e-30)
    return np.abs(a - b).max() / denom


# ---------------------------------------------------------------------------------------------
# Tri-plane activations (precision mode 1, mnc_b200.dense.Tri): with xs = value * 2^exp,
#   h = fp16(xs),  l = e4m3((xs - h) * 2^6),  c = e4m3(xs * 2^-5)   (all saturating)
# The GEMM reads Xh.Wh + Xl.Wc + Xc.Wl, so a wrong l or c plane costs only ~2^-11 of accuracy in
# the next layer and no end-to-end comparison sees it: check_tri checks each plane on its own.
def _e4m3_f64(x):
    """float64 value of the saturating e4m3 rounding of float64 x (torch: the e4m3 grid is exact
    in float32 and |x| is far from the float32 rounding of any e4m3 midpoint where it matters)."""
    import torch
    return x.clamp(-448.0, 448.0).float().to(torch.float8_e4m3fn).double()


def _e4m3_half_step(v):
    """Half the e4m3 quantum at |v| (v an e4m3 value, float64): normal binades have 3 mantissa
    bits, subnormals a quantum of 2^-9; the quantum of the next binade up is used at a power of
    two, which covers values that rounded up into it."""
    import torch
    a = v.abs()
    e = torch.floor(torch.log2(a.clamp_min(2.0 ** -6)))
    return torch.exp2(e - 3.0) / 2.0


def _f16_ulp(h):
    """fp16 ulp of each h (float64 tensor of fp16 values): 2^(E-10), 2^-24 for subnormals."""
    import torch
    a = h.abs()
    e = torch.floor(torch.log2(a.clamp_min(2.0 ** -14)))
    return torch.exp2(e - 10.0)


def tri_rounding(ref, exp):
    """Bound on |decoded - value| of a correctly written activation Tri, with a factor 2 of slack:
    the e4m3 rounding of the residual costs at most 2^-15 * |value| (normal residuals) or
    2^-16 * 2^-exp (subnormal ones).  Above |value * 2^exp| = 2^14 the residual (up to half an fp16
    ulp of 16) saturates at 448 / 64 = 7: there the value is only good to 2^-11 relative."""
    import torch
    a = ref.abs()
    rel = torch.where(a * 2.0 ** exp >= 2.0 ** 14, torch.full_like(a, 2.0 ** -11), torch.full_like(a, 2.0 ** -14))
    return a * rel + 2.0 ** (-15 - exp)


def check_tri(t, ref, exp, bound, region=None, before=None, what="tri"):
    """Assert that the activation Tri `t` holds `ref` (float64) written with exponent `exp`.

    t       dense.Tri whose planes cover the whole buffer (written region and padding).
    ref     float64 values of t[region] (any device; compared on the CPU).
    bound   allowed |decoded - ref|, a number or a tensor broadcastable to ref.
    region  index into t's planes of the written part (None: all of it).
    before  a clone of t taken before the launch: every byte outside `region` must be unchanged,
            in all three planes.

    Checks, element by element over the region:
    1. value: |(h + l/64) * 2^-exp - ref| <= bound;
    2. h is the fp16 rounding of v = h + l/64: |l|/64 <= ulp(h)/2, and <= ulp(h)/4 when h is a
       power of two and l points into the binade below.  64 * ulp/2 is a power of two, so the
       e4m3 rounding of the residual can never cross the bound: this holds exactly.  It also holds
       in the fp16 subnormal range (l is 0 there) and where h saturates (l saturates at 448 <
       64 * ulp/2);
    3. c is the e4m3 rounding of v / 32.  v carries the pre-rounding value xs only to within the
       e4m3 rounding of l (half its quantum, / 64; or 2^-14 * |v| if larger), so c may be the
       rounding of any value in that interval: where v lies within it of an e4m3 midpoint, either
       neighbour is accepted.  Where l saturated (|xs| >= 2^14) c saturates too (|xs|/32 > 448).
    The sign bit of a zero l or c is not checked (the sign of a zero residual is not defined by
    the format)."""
    import torch
    assert t.exp == exp, "%s: exponent %d, expected %d" % (what, t.exp, exp)
    h_all = t.h.detach().cpu()
    l_all = t.l.detach().cpu()
    c_all = t.c.detach().cpu()
    if region is None:
        mask = torch.ones(h_all.shape, dtype=torch.bool)
    else:
        mask = torch.zeros(h_all.shape, dtype=torch.bool)
        mask[region] = True
    if before is not None:
        out = ~mask
        for name, now, old in (("h", h_all.view(torch.int16), before.h.detach().cpu().view(torch.int16)),
                               ("l", l_all, before.l.detach().cpu()), ("c", c_all, before.c.detach().cpu())):
            bad = (now != old) & out
            assert not bool(bad.any()), "%s: %d padding bytes of plane %s overwritten, first at %s" % (
                what, int(bad.sum()), name, tuple(bad.nonzero()[0].tolist()))
    h = h_all[mask].double()
    l = l_all[mask].view(torch.float8_e4m3fn).double()
    c = c_all[mask].view(torch.float8_e4m3fn).double()
    ref = ref.detach().cpu().double().reshape(-1)
    assert ref.numel() == h.numel(), "%s: ref has %d elements, region %d" % (what, ref.numel(), h.numel())
    assert bool(torch.isfinite(h).all() & torch.isfinite(l).all() & torch.isfinite(c).all()), \
        "%s: non-finite plane values" % what

    def fail(name, bad, detail):
        i = int(bad.nonzero()[0])
        raise AssertionError("%s: %s fails at %d of %d elements; first (flat %d): h=%r l=%r c=%r ref=%r %s"
                             % (what, name, int(bad.sum()), bad.numel(), i, float(h[i]), float(l[i]),
                                float(c[i]), float(ref[i]), detail(i)))

    v = h + l / 64.0                                   # exact in float64
    err = (v * 2.0 ** -exp - ref).abs()
    bnd = torch.as_tensor(bound, dtype=torch.float64)
    bnd = bnd.detach().cpu().reshape(-1) if bnd.dim() else bnd
    bad = err > bnd
    if bool(bad.any()):
        fail("value", bad, lambda i: "|err|=%r bound=%r" % (float(err[i]), float(bnd if bnd.dim() == 0 else bnd[i])))
    ulp = _f16_ulp(h)
    pow2 = (h.abs() >= 2.0 ** -13) & (torch.frexp(h)[0].abs() == 0.5)
    inward = pow2 & (l * h < 0)
    lim = torch.where(inward, ulp / 4.0, ulp / 2.0)
    bad = l.abs() / 64.0 > lim
    if bool(bad.any()):
        fail("h = fp16(value)", bad, lambda i: "|l|/64=%r > %r" % (float(l[i].abs() / 64), float(lim[i])))
    unc = torch.maximum(_e4m3_half_step(l) / 64.0, v.abs() * 2.0 ** -14)
    unc = torch.where(l.abs() == 448.0, ulp, unc)
    lo, hi = _e4m3_f64((v - unc) / 32.0), _e4m3_f64((v + unc) / 32.0)
    bad = (c < lo) | (c > hi)
    if bool(bad.any()):
        fail("c = e4m3(value / 32)", bad, lambda i: "c in [%r, %r] expected" % (float(lo[i]), float(hi[i])))


# ---------------------------------------------------------------------------------------------
# Test-only HDF5 assembler (superblock v0, old-style groups, contiguous float32 datasets): builds
# files with NESTED groups and multi-node group B-trees byte by byte from the file-format
# specification, to exercise mnc_b200/hdf5_min.py beyond the flat files the reference ships.
def write_h5_tree(path, tree):
    """tree: {name: ndarray | subtree}.  Datasets are written as contiguous little-endian float32."""
    import struct
    UNDEF = 0xFFFFFFFFFFFFFFFF
    buf = bytearray(b"\x00" * 96)          # superblock v0 (56 bytes) + root symbol-table entry (40)

    def alloc(n):
        while len(buf) % 8:
            buf.append(0)
        off = len(buf)
        buf.extend(b"\x00" * n)
        return off

    def put(off, data):
        buf[off:off + len(data)] = data

    def msg(mtype, body):
        body = bytes(body) + b"\x00" * (-len(body) % 8)
        return struct.pack("<HHB3x", mtype, len(body), 0) + body

    def header(msgs):
        body = b"".join(msgs)
        off = alloc(16 + len(body))
        put(off, struct.pack("<BBHII4x", 1, 0, len(msgs), 1, len(body)) + body)
        return off

    def dataset(arr):
        arr = np.ascontiguousarray(arr, dtype="<f4")
        data_off = alloc(arr.nbytes)
        put(data_off, arr.tobytes())
        space = struct.pack("<BBB5x", 1, arr.ndim, 0) + b"".join(struct.pack("<Q", d) for d in arr.shape)
        dtype = struct.pack("<BBBBI", 0x11, 0x20, 0x1F, 0x00, 4) + struct.pack("<HHBBBBI", 0, 32, 23, 8, 0, 23, 127)
        layout = struct.pack("<BBQQ", 3, 1, data_off, arr.nbytes)
        return header([msg(0x01, space), msg(0x03, dtype), msg(0x08, layout)])

    def group(sub):
        children = []
        for name in sorted(sub):           # group B-trees keep names in order
            v = sub[name]
            children.append((name, group(v)[0] if isinstance(v, dict) else dataset(v)))
        heap_data = bytearray(b"\x00" * 8)
        name_off = {}
        for name, _ in children:
            name_off[name] = len(heap_data)
            raw = name.encode() + b"\x00"
            heap_data.extend(raw + b"\x00" * (-len(raw) % 8))
        hd = alloc(len(heap_data))
        put(hd, heap_data)
        heap = alloc(32)
        put(heap, b"HEAP" + struct.pack("<B3xQQQ", 0, len(heap_data), UNDEF, hd))
        snods = []
        for s in range(0, max(len(children), 1), 8):       # 2 * leaf K = 8 symbols per node
            part = children[s:s + 8]
            node = alloc(8 + 8 * 40)
            ent = b"".join(struct.pack("<QQII16x", name_off[n], a, 0, 0) for n, a in part)
            put(node, b"SNOD" + struct.pack("<BBH", 1, 0, len(part)) + ent)
            snods.append((node, name_off[part[-1][0]] if part else 0))
        tree_off = alloc(24 + (2 * 32 + 1) * 8 + 2 * 32 * 8)
        body = b"TREE" + struct.pack("<BBHQQ", 0, 0, len(snods), UNDEF, UNDEF) + struct.pack("<Q", 0)
        for node, last_name in snods:
            body += struct.pack("<QQ", node, last_name)
        put(tree_off, body)
        return header([msg(0x11, struct.pack("<QQ", tree_off, heap))]), tree_off, heap

    root, btree, heap = group(tree)
    put(0, b"\x89HDF\r\n\x1a\n" + struct.pack("<BBBBBBBBHHI", 0, 0, 0, 0, 0, 8, 8, 0, 4, 16, 0) +
        struct.pack("<QQQQ", 0, UNDEF, len(buf), UNDEF) +
        struct.pack("<QQII", 0, root, 1, 0) + struct.pack("<QQ", btree, heap))
    with open(path, "wb") as f:
        f.write(bytes(buf))
