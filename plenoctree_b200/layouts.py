"""numpy mirrors of the shared-memory operand layouts of csrc/common.cuh.

Used by the tests to build operand images and to check the device pack kernel; kept next to the
product code because the layouts are part of the kernel contract.
"""
import numpy as np

TILE_M = 128
A_CHUNK_BYTES = 128 * 128
WSLOT_BYTES = 256 * 64


def a_tile_offset(row, col):
    """byte offset of fp16 element (row, col) in a K-major SW128 activation tile image."""
    row = np.asarray(row)
    col = np.asarray(col)
    return ((col >> 6) * A_CHUNK_BYTES + row * 128 + ((((col >> 3) & 7) ^ (row & 7)) << 4)
            + (col & 7) * 2)


def w_slot_offset(row, k):
    """byte offset of fp16 element (row, k<32) in a K-major SW64 weight slot image."""
    row = np.asarray(row)
    k = np.asarray(k)
    return row * 64 + ((((k >> 3) & 3) ^ ((row >> 1) & 3)) << 4) + (k & 7) * 2


def pack_a_tile(mat):
    """[128, 64*n] float -> uint8 image (fp16, SW128)."""
    rows, cols = mat.shape
    assert rows == 128 and cols % 64 == 0
    img = np.zeros(A_CHUNK_BYTES * (cols // 64), dtype=np.uint8)
    h = mat.astype(np.float16).view(np.uint16)
    r, c = np.meshgrid(np.arange(rows), np.arange(cols), indexing="ij")
    off = a_tile_offset(r, c)
    img16 = img.view(np.uint16)
    img16[off // 2] = h
    return img


def unpack_a_tile(img, cols):
    r, c = np.meshgrid(np.arange(128), np.arange(cols), indexing="ij")
    off = a_tile_offset(r, c)
    return img.view(np.uint16)[off // 2].view(np.float16).astype(np.float32)


def t_tile_offset(row, col):
    """byte offset of fp16 element (row, col) in a "T" tile image: [32-row group][8-column unit]
    [row in group][16 B].  mlp_fwd writes the saved h_l tiles in this order (one coalesced 512 B
    store per warp instruction); read MN-major by the tensor
    cores it is the canonical no-swizzle layout with 128 B core matrices (8 rows x 8 columns):
    LBO (next 8 rows) = 128 B, SBO (next 8 columns) = 512 B."""
    row = np.asarray(row)
    col = np.asarray(col)
    return (row >> 5) * 16384 + (col >> 3) * 512 + (row & 31) * 16 + (col & 7) * 2


def pack_t_tile(mat):
    """[128, 256] float -> uint8 image (fp16, T layout)."""
    rows, cols = mat.shape
    assert rows == 128 and cols == 256
    img = np.zeros(rows * cols * 2, dtype=np.uint8)
    r, c = np.meshgrid(np.arange(rows), np.arange(cols), indexing="ij")
    img.view(np.uint16)[t_tile_offset(r, c) // 2] = mat.astype(np.float16).view(np.uint16)
    return img


def unpack_t_tile(img):
    r, c = np.meshgrid(np.arange(128), np.arange(256), indexing="ij")
    return img.view(np.uint16)[t_tile_offset(r, c) // 2].view(np.float16).astype(np.float32)


def pack_w_slot(mat):
    """[rows, 32] float -> uint8 image (fp16, SW64)."""
    rows, k = mat.shape
    assert k == 32 and rows % 8 == 0
    img = np.zeros(rows * 64, dtype=np.uint8)
    r, c = np.meshgrid(np.arange(rows), np.arange(32), indexing="ij")
    img.view(np.uint16)[w_slot_offset(r, c) // 2] = mat.astype(np.float16).view(np.uint16)
    return img


# ---- flat parameter layout / packed image geometry (mirrors csrc/kernels.h, pack.cu) ---------
def K_of(sh_deg):
    return 1 if sh_deg < 0 else (sh_deg + 1) ** 2


def heads_width(K):
    return (1 + 3 * K + 15) // 16 * 16


def fwd_has_bias_slot(l):
    return not (l == 0 or l == 5)


def fwd_slots_of_layer(l):
    return 2 if l == 0 else (10 if l == 5 else 9)


ENC_DIM = 63      # posenc width of the default encoder (0, 10); columns [W, 63) of the posenc tile are 0, 63 is 1
POSENC_MAX_DEG = 10


def posenc_width(posenc=None):
    """W = 3 + 6 (max_deg - min_deg) of the point encoder (min_deg, max_deg, legacy); None = (0, 10) -> 63."""
    if posenc is None:
        return ENC_DIM
    return 3 + 6 * (int(posenc[1]) - int(posenc[0]))


def posenc_valid(posenc):
    """the encoders the kernels take: 0 <= min_deg <= max_deg <= 10 (mirrors kernels.h posenc_valid)."""
    mn, mx = int(posenc[0]), int(posenc[1])
    return 0 <= mn <= mx <= POSENC_MAX_DEG


def layer_dims(K, W=ENC_DIM):
    """(in, out) of Dense_0..Dense_9 for K SH coefficients and posenc width W: Dense_0 [W, 256], Dense_5 [256 + W, 256]
    (rows [h4 | posenc])."""
    dims = []
    for i in range(10):
        cin = W if i == 0 else (256 + W if i == 5 else 256)
        cout = 256 if i < 8 else (1 if i == 8 else 3 * K)
        dims.append((cin, cout))
    return dims


def flat_offsets(K, W=ENC_DIM):
    w_off, b_off, off = [], [], 0
    for cin, cout in layer_dims(K, W):
        w_off.append(off)
        off += cin * cout
        b_off.append(off)
        off += cout
    return w_off, b_off, off


def blob_layout(K):
    NH = heads_width(K)
    up = lambda x: (x + 1023) // 1024 * 1024
    fwd = 66 * 16384 + 9 * NH * 64
    bwd = ((NH + 31) // 32 + 56) * 16384
    w_hi = 0
    w_lo = up(w_hi + fwd)
    wt_hi = up(w_lo + fwd)
    total = up(wt_hi + bwd)
    return dict(w_hi=w_hi, w_lo=w_lo, wt_hi=wt_hi, total=total, fwd_bytes=fwd, bwd_bytes=bwd, NH=NH)


def heads_matrix(flat, K, W=ENC_DIM):
    """packed heads weight [256 in, NH] and bias [NH] in kernel column order [sigma, (k,c)...]."""
    w_off, b_off, _ = flat_offsets(K, W)
    NH = heads_width(K)
    W8 = flat[w_off[8]:w_off[8] + 256].reshape(256, 1)
    W9 = flat[w_off[9]:w_off[9] + 256 * 3 * K].reshape(256, 3 * K)
    b8 = flat[b_off[8]:b_off[8] + 1]
    b9 = flat[b_off[9]:b_off[9] + 3 * K]
    Wh = np.zeros((256, NH), np.float32)
    bh = np.zeros(NH, np.float32)
    Wh[:, 0] = W8[:, 0]
    bh[0] = b8[0]
    for k in range(K):
        for c in range(3):
            Wh[:, 1 + 3 * k + c] = W9[:, c * K + k]
            bh[1 + 3 * k + c] = b9[c * K + k]
    return Wh, bh


def heads_column(K, o):
    """packed heads column of Dense_9 output o (reference channel-major order c*K + k)."""
    c, k = divmod(o, K)
    return 1 + 3 * k + c


def pack_reference(flat, sh_deg, posenc=None):
    """numpy model of pack.cu: returns dict of uint8 images w_hi, w_lo, wt_hi.  posenc = (min_deg, max_deg, legacy)
    of the model (None: the default); the images keep their size, with rows [W, 63) of the posenc slots zero."""
    K = K_of(sh_deg)
    W = posenc_width(posenc)
    L = blob_layout(K)
    NH = L["NH"]
    w_off, b_off, total = flat_offsets(K, W)
    flat = np.asarray(flat, np.float32)
    assert flat.size == total
    dims = layer_dims(K, W)
    w_hi = np.zeros(L["fwd_bytes"], np.uint8)
    w_lo = np.zeros(L["fwd_bytes"], np.uint8)
    wt_hi = np.zeros(L["bwd_bytes"], np.uint8)

    def hilo(m):
        hi = m.astype(np.float16)
        lo = (m - hi.astype(np.float32)).astype(np.float16)
        return hi, lo

    slot = 0
    for l in range(8):
        cin = dims[l][0]
        Wl = flat[w_off[l]:w_off[l] + cin * 256].reshape(cin, 256)  # [in, out]
        if not fwd_has_bias_slot(l):
            # layers 0 / 5: the K rows follow the posenc tile's 64 columns, the bias on its constant column 63
            h = cin - W                            # h4 rows before the posenc rows (layer 5)
            full = np.zeros((h + 64, 256), np.float32)
            full[:cin] = Wl
            full[h + 63] = flat[b_off[l]:b_off[l] + 256]
            Wl = full
        bias_l = flat[b_off[l]:b_off[l] + 256]
        for j in range(fwd_slots_of_layer(l)):
            blk = np.zeros((256, 32), np.float32)  # [out row, k]
            if fwd_has_bias_slot(l) and j == 8:
                blk[:, 31] = bias_l                # bias slot: multiplied by posenc column 63 (= 1)
            else:
                blk[:, :] = Wl[32 * j:32 * j + 32, :].T
            hi, lo = hilo(blk)
            w_hi[slot * 16384:(slot + 1) * 16384] = pack_w_slot(hi)
            w_lo[slot * 16384:(slot + 1) * 16384] = pack_w_slot(lo)
            slot += 1
    Wh, bh = heads_matrix(flat, K, W)
    base = 66 * 16384
    for j in range(9):
        if j < 8:
            blk = Wh[32 * j:32 * j + 32, :].T  # [NH, 32]
        else:
            blk = np.zeros((NH, 32), np.float32)
            blk[:, 31] = bh
        hi, lo = hilo(blk)
        w_hi[base + j * NH * 64: base + (j + 1) * NH * 64] = pack_w_slot(hi)
        w_lo[base + j * NH * 64: base + (j + 1) * NH * 64] = pack_w_slot(lo)
    # dgrad images: rows = in feature, k = out feature
    hs = (NH + 31) // 32
    slot = 0
    for j in range(hs):
        blk = np.zeros((256, 32), np.float32)
        kn = max(0, min(32, NH - 32 * j))
        blk[:, :kn] = Wh[:, 32 * j:32 * j + kn]
        wt_hi[slot * 16384:(slot + 1) * 16384] = pack_w_slot(blk)
        slot += 1
    for l in range(7, 0, -1):
        cin = dims[l][0]
        Wl = flat[w_off[l]:w_off[l] + cin * 256].reshape(cin, 256)[:256]  # [in(256), out]
        for j in range(8):
            wt_hi[slot * 16384:(slot + 1) * 16384] = pack_w_slot(Wl[:, 32 * j:32 * j + 32])
            slot += 1
    return dict(w_hi=w_hi, w_lo=w_lo, wt_hi=wt_hi)


# ---- training workspace (mirrors carve() in csrc/pipeline.cu) ------------------------------------------------------
# Every intermediate of pob_loss_and_grad stays in the caller's workspace, so that a test can check each kernel of the
# training chain on its own, with the GPU's own inputs.  The decoders below turn those bytes into torch tensors on the
# workspace's device (the production step's tiles are far too large for numpy).
NUM_TRUNK = 8
A_TILE_BYTES = 4 * A_CHUNK_BYTES          # [128 x 256] fp16
E_TILE_BYTES = A_CHUNK_BYTES              # [128 x 64] fp16
DO_TILE_BYTES = 2 * A_CHUNK_BYTES         # [128 x 128] fp16
WG_MAX_CTAS = 160
WG_PARTIAL_FLOATS = 65536 + 256


def padded_rows(M):
    """rows of every per-sample training array: a multiple of four 128-row tiles (common.cuh: padded_rows)."""
    return (M + 511) // 512 * 512


def bwd_image_bytes(K):
    """bytes of one dgrad weight image (kernels.h: bwd_image_bytes)."""
    return blob_layout(K)["bwd_bytes"]


def train_workspace_views(cfg, n_rays, sparsity_on, training=True, precision=1):
    """Byte layout of the training workspace of `cfg` (a RenderConfig or anything with its fields) for a
    pob_loss_and_grad call over `n_rays` rays; `sparsity_on` = the call carries the sparsity points (weight > 0).

    Returns dict(total=bytes, partials=[offsets], levels=[...]) with one entry per level (coarse, then fine when
    num_fine_samples > 0).  Each level holds (offset, shape) pairs for z, rgbs, weights, comp, disp, acc (float32;
    rgbs and G as [rows, 4]), G, H [tiles, 8, 64 KB], E [tiles, 16 KB], DZ [tiles, 8, 64 KB], DO [tiles, 32 KB]
    (uint8 tile images), mask [8, rows, 8] and progress [tiles] (uint32 words), sized for this call, plus the call's
    row counts: N samples per ray, M_rays, M (with the sparsity rows, which ride behind the rays of the last level),
    rows (= padded_rows(M)) and tiles.  Buffers are carved for cfg.max_rays; the mask's per-layer stride is the call's
    padded row count.

    training=False: the render workspace of pob_render_rays (pob_workspace_bytes(cfg, 0)).  Each level then holds
    only z, rgbs, weights, comp, disp and acc, no sparsity rows, and partials is empty.

    precision=3 (POB_PREC_FP16X3): the workspace of pob_loss_and_grad_prec at fp16x3
    (pob_train_workspace_bytes(cfg, 3)): the fp16 views, plus per level the residual images H_lo, E_lo, DZ_lo, DO_lo
    (shaped like H, E, DZ, DO), partials_x3 = [[mlp 0 pass 1, pass 2], [mlp 1 ...]] and wt_lo = [mlp 0, mlp 1]
    (offset, bytes) of the residual dgrad weight images."""
    R = int(cfg.max_rays)
    nc, nf, nsp = int(cfg.num_coarse_samples), int(cfg.num_fine_samples), int(cfg.sparsity_npoints)
    Ns = [nc, nc + nf if nf > 0 else 0]
    last = 1 if nf > 0 else 0
    off = 0
    levels = []
    caps = [0, 0]      # tiles carved per level

    def take(nbytes):
        nonlocal off
        o = off
        off += (nbytes + 1023) // 1024 * 1024
        return o

    for lv in range(2):
        Mr_cap = R * Ns[lv]
        M_cap = Mr_cap + (nsp if (training and lv == last) else 0)
        tiles_cap = caps[lv] = padded_rows(M_cap) // TILE_M
        if Mr_cap == 0:
            continue
        N = Ns[lv]
        M_rays = n_rays * N
        M = M_rays + (nsp if (training and lv == last and sparsity_on) else 0)
        rows = padded_rows(M)
        tiles = rows // TILE_M
        v = dict(N=N, M_rays=M_rays, M=M, rows=rows, tiles=tiles)
        v["z"] = (take(4 * Mr_cap), (n_rays, N))
        v["rgbs"] = (take(16 * M_cap), (M, 4))
        v["weights"] = (take(4 * Mr_cap), (n_rays, N))
        v["comp"] = (take(12 * R), (n_rays, 3))
        v["disp"] = (take(4 * R), (n_rays,))
        v["acc"] = (take(4 * R), (n_rays,))
        if not training:
            levels.append(v)
            continue
        v["G"] = (take(16 * M_cap), (M, 4))
        v["H"] = (take(tiles_cap * NUM_TRUNK * A_TILE_BYTES), (tiles, NUM_TRUNK, A_TILE_BYTES))
        v["E"] = (take(tiles_cap * E_TILE_BYTES), (tiles, E_TILE_BYTES))
        v["DZ"] = (take(tiles_cap * NUM_TRUNK * A_TILE_BYTES), (tiles, NUM_TRUNK, A_TILE_BYTES))
        v["DO"] = (take(tiles_cap * DO_TILE_BYTES), (tiles, DO_TILE_BYTES))
        v["mask"] = (take(NUM_TRUNK * tiles_cap * TILE_M * 8 * 4), (NUM_TRUNK, rows, 8))
        levels.append(v)
    if not training:
        return dict(total=off, levels=levels, partials=[])
    partials = [take(4 * WG_MAX_CTAS * WG_PARTIAL_FLOATS) for _ in range(2)]
    progress = take(4 * sum(caps))   # mlp_bwd -> mlp_wgrad progress counters, level 0's tiles then level 1's
    for v, first in zip(levels, (0, caps[0])):
        v["progress"] = (progress + 4 * first, (v["tiles"],))
    if precision != 3:
        return dict(total=off, levels=levels, partials=partials)
    for v, cap in zip(levels, caps):
        for name, per_tile in (("H", NUM_TRUNK * A_TILE_BYTES), ("E", E_TILE_BYTES), ("DZ", NUM_TRUNK * A_TILE_BYTES),
                               ("DO", DO_TILE_BYTES)):
            v[name + "_lo"] = (take(cap * per_tile), v[name][1])
    partials_x3 = [[take(4 * WG_MAX_CTAS * WG_PARTIAL_FLOATS) for _ in range(2)] for _ in range(2)]
    nb = bwd_image_bytes(K_of(int(cfg.sh_deg)))
    wt_lo = [(take(nb), nb) for _ in range(2)]
    return dict(total=off, levels=levels, partials=partials, partials_x3=partials_x3, wt_lo=wt_lo)


_VIEW_DTYPES = dict(z="float32", rgbs="float32", weights="float32", comp="float32", disp="float32", acc="float32",
                    G="float32", H="uint8", E="uint8", DZ="uint8", DO="uint8", mask="int32",
                    progress="int32", H_lo="uint8", E_lo="uint8", DZ_lo="uint8", DO_lo="uint8")


def workspace_view(ws, level, name):
    """torch view of buffer `name` of one level (an entry of train_workspace_views()["levels"]) in the uint8
    workspace tensor `ws`."""
    import torch
    off, shape = level[name]
    dt = getattr(torch, _VIEW_DTYPES[name])
    n = int(np.prod(shape)) * torch.empty((), dtype=dt).element_size()
    return ws[off:off + n].view(dt).view(shape)


_GATHER = {}


def _gather_index(kind, device):
    """int64 [128 * cols] index of fp16 element (row, col) of one tile image, row-major over (row, col)."""
    import torch
    key = (kind, str(device))
    if key not in _GATHER:
        cols = {"T": 256, "A256": 256, "A128": 128, "A64": 64}[kind]
        r, c = np.meshgrid(np.arange(TILE_M), np.arange(cols), indexing="ij")
        off = t_tile_offset(r, c) if kind == "T" else a_tile_offset(r, c)
        _GATHER[key] = torch.from_numpy((off // 2).reshape(-1).astype(np.int64)).to(device)
    return _GATHER[key]


def _decode(tiles_u8, kind, cols):
    import torch
    T = tiles_u8.shape[0]
    u16 = tiles_u8.reshape(T, -1).view(torch.int16)
    return u16[:, _gather_index(kind, tiles_u8.device)].view(torch.float16).reshape(T * TILE_M, cols)


def decode_h(H, layer):
    """H [tiles, 8, 64 KB] (T layout) -> fp16 h_layer [tiles * 128, 256]."""
    return _decode(H[:, layer].contiguous(), "T", 256)


def decode_dz(DZ, layer):
    """DZ [tiles, 8, 64 KB] (SW128) -> fp16 dz_layer [tiles * 128, 256]."""
    return _decode(DZ[:, layer].contiguous(), "A256", 256)


def decode_e(E):
    """E [tiles, 16 KB] (SW128) -> fp16 posenc [tiles * 128, 64] (columns [W, 63) = 0, column 63 = 1)."""
    return _decode(E, "A64", 64)


def decode_do(DO):
    """DO [tiles, 32 KB] (SW128) -> fp16 dO [tiles * 128, 128] (packed heads columns: sigma, then 1 + 3k + c)."""
    return _decode(DO, "A128", 128)


def mask_bit_of_column():
    """bit of column j (0..31) inside its mask word: column 2k -> bit 15 - k, column 2k + 1 -> bit 31 - k."""
    j = np.arange(32)
    return np.where(j % 2 == 0, 15 - j // 2, 31 - j // 2)


def decode_mask(words):
    """mask words [..., rows, 8] (int32 or uint32) -> bool [..., rows, 256]; word c covers columns 32c..32c+31."""
    import torch
    w = torch.as_tensor(words)
    w = (w.to(torch.int64) & 0xFFFFFFFF)
    col = np.arange(256)
    word = torch.from_numpy(col // 32).to(w.device)
    bit = torch.from_numpy(mask_bit_of_column()[col % 32].astype(np.int64)).to(w.device)
    return ((w[..., word] >> bit) & 1).bool()


def encode_mask_reference(h):
    """numpy model of mlp_fwd's mask store: h [rows, 256] -> uint32 words [rows, 8].  Per word, the sixteen fp16 pairs
    (2k, 2k+1) are shifted in from the left, one per step: each step shifts the word left by one and adds
    (h[2k] != 0) + ((h[2k+1] != 0) << 16)."""
    nz = (np.asarray(h) != 0)
    rows = nz.shape[0]
    out = np.zeros((rows, 8), np.uint32)
    for c in range(8):
        m = np.zeros(rows, np.uint32)
        for k in range(16):
            pair = nz[:, 32 * c + 2 * k].astype(np.uint32) + (nz[:, 32 * c + 2 * k + 1].astype(np.uint32) << 16)
            m = (m << np.uint32(1)) + pair
        out[:, c] = m
    return out
