"""Shared by the carrier-tokenizer kernel tests (test_glue_kernels_gpu.py, test_detection_kernels_gpu.py) and the
detection-plan tests: the scattered problem layout of the TokenInitializer kernels, and the seeded sweep of DETR
training input sizes."""
import torch


def token_init_problem(g, B, Hp, Wp, C, kh, kw, sh, sw):
    """A B x C x Hp x Wp map stored as scattered rows of xs (row stride C + 4, 17 spare rows): pix_map sends pixel
    (b, y, x) to its row, about 15 % of the pixels are -1 (the zero padding pixels of an any-res map); ct_rows sends
    each of the B * oh * ow carrier slots to a distinct row of a buffer with 9 spare rows. xmap is the fp64 NCHW map
    the kernels read."""
    oh, ow = (Hp - kh) // sh + 1, (Wp - kw) // sw + 1
    npix = B * Hp * Wp
    total = npix + 17
    pix_map = torch.randperm(total, device="cuda", generator=g)[:npix].int()
    pad = torch.rand(npix, device="cuda", generator=g) < 0.15        # padding pixels of an any-res map read as zero
    pix_map[pad] = -1
    xs = torch.randn(total, C + 4, device="cuda", generator=g)
    xmap = torch.zeros(npix, C, dtype=torch.float64, device="cuda")
    xmap[~pad] = xs[pix_map[~pad].long(), :C].double()
    xmap = xmap.view(B, Hp, Wp, C).permute(0, 3, 1, 2)
    w = torch.randn(C, 1, 3, 3, device="cuda", generator=g) * 0.3
    bias = torch.randn(C, device="cuda", generator=g) * 0.1
    nct = B * oh * ow
    ct_rows = (torch.randperm(nct + 9, device="cuda", generator=g)[:nct]).int()
    return dict(oh=oh, ow=ow, npix=npix, total=total, pix_map=pix_map, pad=pad, xs=xs, xmap=xmap, w=w, bias=bias,
                nct=nct, ct_rows=ct_rows)


def detr_shapes(n, seed=0):
    """(H, W) of n distinct batches of DETR's multi-scale training augmentation: short side from 480..800 in steps of
    32, long side capped at 1333, a random aspect ratio per batch (rounded to multiples of 4 to keep the sweep short)"""
    g = torch.Generator().manual_seed(seed)
    shapes = []
    while len(shapes) < n:
        s = 480 + 32 * int(torch.randint(0, 11, (1,), generator=g))
        r = 1.0 + float(torch.rand(1, generator=g)) * 0.8
        long = min(int(s * r), 1333)
        hw = (s // 4 * 4, long // 4 * 4) if torch.rand(1, generator=g) < 0.5 else (long // 4 * 4, s // 4 * 4)
        if hw not in shapes:
            shapes.append(hw)
    return shapes


def level_sizes(H, W):
    """the input map of each of the four levels of an H x W image (stem: two stride-2 convolutions; a stride-2
    Downsample between levels), as the detection plans size them"""
    h, w = (H + 1) // 2, (W + 1) // 2
    sizes = [((h + 1) // 2, (w + 1) // 2)]
    for _ in range(3):
        sizes.append(((sizes[-1][0] + 1) // 2, (sizes[-1][1] + 1) // 2))
    return sizes
