"""TrivialAugment Wide, AutoAugment and random erasing of training batches (``--auto-augment ta_wide|imagenet|cifar10|svhn``,
``--random-erase P``).

The semantics are torchvision 0.26's, applied per sample as the classification recipe's ``ClassificationPresetTrain`` does:
``transforms.v2.TrivialAugmentWide(interpolation=BILINEAR)`` or ``transforms.v2.AutoAugment(policy, interpolation=BILINEAR)``
on the uint8 crop, then the normalisation, then ``transforms.v2.RandomErasing(p, scale=(0.02, 0.33), ratio=(0.3, 3.3),
value=0)`` on the normalised tensor.

On the GPU one ``augment_normalize`` call (``csrc/augment.cu``; two launches for two ops) does all three for the whole batch
and returns what ``normalize_nhwc`` returns: the draws of a batch are encoded on the host into a pinned float32 table that
travels to the device with the batch, ``[n, AUG_PRM]`` for TrivialAugment Wide's one op per sample and ``[n, AUG_CHAIN_PRM]``
for an AutoAugment sub-policy's two ops, the second applied to the first's output.  On the CPU,
:meth:`BatchAugment.reference_apply` runs torchvision's own functional ops
per sample; it is also the reference of the GPU tests.
"""
from __future__ import annotations

import functools
import math
from typing import Optional

import numpy as np
import torch

AUG_PRM = 16                    # columns of the parameter table (kAugPrm in csrc/host.h)
AUG_CHAIN_PRM = 32              # columns of a two-op table (kAugChainPrm): op B's code and parameters in 16..22
COL_B = 16                      # op B's first column; its op index and signed magnitude are in COL_B + 7, COL_B + 8
AUTOAUGMENT_POLICIES = ("imagenet", "cifar10", "svhn")
AA_NUM_BINS = 10                # AutoAugment's magnitude tables have 10 entries
AUG_MAX_PIXELS = 65793          # kAugMaxPixels: 255 H W < 2^24, so Contrast's float32 mean is exact in torchvision's order
NUM_BINS = 31
ERASE_SCALE = (0.02, 0.33)
ERASE_RATIO = (0.3, 3.3)
STREAM_ID = 0x61756721          # the fourth word of the draw stream's key: BatchMix keys its stream with three

# the kernel's op codes (AugOp in csrc/augment.cu)
K_IDENTITY, K_AFFINE, K_ROT90, K_BRIGHTNESS, K_COLOR, K_CONTRAST, K_SHARPNESS, K_POSTERIZE, K_SOLARIZE, K_AUTOCONTRAST, K_EQUALIZE, \
    K_INVERT = range(12)


@functools.lru_cache(maxsize=None)
def _policy():
    from torchvision.transforms import InterpolationMode
    from torchvision.transforms.v2 import TrivialAugmentWide
    return TrivialAugmentWide(num_magnitude_bins=NUM_BINS, interpolation=InterpolationMode.BILINEAR)


@functools.lru_cache(maxsize=None)
def _aa_policy(policy: str):
    from torchvision.transforms import AutoAugmentPolicy, InterpolationMode
    from torchvision.transforms.v2 import AutoAugment
    return AutoAugment(AutoAugmentPolicy(policy), interpolation=InterpolationMode.BILINEAR)


def op_names():
    """The 14 ops in the order of torchvision's ``TrivialAugmentWide._AUGMENTATION_SPACE``."""
    return tuple(_policy()._AUGMENTATION_SPACE.keys())


def chain_names():
    """The op index space of the tables' reference columns: :func:`op_names` and AutoAugment's ``Invert``."""
    return op_names() + ("Invert",)


def sub_policies(policy: str):
    """AutoAugment's 25 sub-policies of ``policy``, ``((name, p, magnitude_idx), (name, p, magnitude_idx))``, as
    torchvision's own ``AutoAugment`` object holds them."""
    return tuple(_aa_policy(policy)._policies)


def aa_magnitude(policy: str, name: str, magnitude_idx, negate: bool, H: int, W: int) -> float:
    """The magnitude AutoAugment applies for an entry: ``_AUGMENTATION_SPACE[name][0](10, H, W)[magnitude_idx]``, negated
    for a signed op when ``negate`` (0.0 for the ops without a table)."""
    fn, signed = _aa_policy(policy)._AUGMENTATION_SPACE[name]
    mags = fn(AA_NUM_BINS, H, W)
    if mags is None:
        return 0.0
    m = float(mags[magnitude_idx])
    return -m if (signed and negate) else m


def magnitude(op: int, bin_: int, negate: bool, H: int, W: int) -> float:
    """The magnitude torchvision applies for op index ``op`` and bin ``bin_``: its own float32 table's value, negated for a
    signed op when ``negate`` (0.0 for the ops without a table)."""
    names = op_names()
    if not (0 <= op < len(names)):
        raise ValueError("op index %r outside [0, %d)" % (op, len(names)))
    if not (0 <= bin_ < NUM_BINS):
        raise ValueError("magnitude bin %r outside [0, %d)" % (bin_, NUM_BINS))
    fn, signed = _policy()._AUGMENTATION_SPACE[names[op]]
    mags = fn(NUM_BINS, H, W)
    if mags is None:
        return 0.0
    m = float(mags[bin_])
    return -m if (signed and negate) else m


def _f32(v: float) -> float:
    return float(np.float32(v))


def _grid_theta(matrix, H: int, W: int):
    """_affine_grid's rescaled theta: the fp32 inverse matrix, each row divided in fp32 by W/2 (x) or H/2 (y)."""
    m = np.asarray(matrix, dtype=np.float32)
    hw, hh = np.float32(0.5 * W), np.float32(0.5 * H)
    return [float(v) for v in (m[0] / hw, m[1] / hw, m[2] / hw, m[3] / hh, m[4] / hh, m[5] / hh)]


@functools.lru_cache(maxsize=65536)
def encode(op: int, bin_: int, negate: bool, H: int, W: int):
    """Kernel code and parameters (prm[0..6]) of one draw, with the scalars rounded as torchvision rounds them."""
    mag = magnitude(op, bin_, negate, H, W)          # raises for an op index or bin out of range
    return op_code(op_names()[op], mag, H, W)


def op_code(name: str, mag: float, H: int, W: int):
    """Kernel code and parameters of op ``name`` at magnitude ``mag`` (as ``_apply_image_or_video_transform`` takes them)
    on an ``H x W`` image, with the scalars rounded as torchvision rounds them."""
    from torchvision.transforms.v2.functional._geometry import _get_inverse_affine_matrix
    if name in ("ShearX", "ShearY", "TranslateX", "TranslateY", "Rotate"):
        # the arguments _apply_image_or_video_transform gives F.affine / F.rotate, turned into affine_image's and
        # rotate_image's center_f, translate and shear
        if name == "Rotate":
            angle = mag % 360
            if angle == 0:
                return (K_IDENTITY,)
            if angle == 180:
                raise ValueError("Rotate by 180 is not in the range of TrivialAugmentWide or AutoAugment")
            if H == W and angle in (90, 270):
                return (K_ROT90, 1 if angle == 90 else 3)
            matrix = _get_inverse_affine_matrix([0.0, 0.0], -angle, [0.0, 0.0], 1.0, [0.0, 0.0])
        elif name in ("ShearX", "ShearY"):
            deg = math.degrees(math.atan(mag))
            shear = [deg, 0.0] if name == "ShearX" else [0.0, deg]
            matrix = _get_inverse_affine_matrix([-W * 0.5, -H * 0.5], 0.0, [0.0, 0.0], 1.0, shear)
        else:
            t = [float(int(mag)), 0.0] if name == "TranslateX" else [0.0, float(int(mag))]
            matrix = _get_inverse_affine_matrix([0.0, 0.0], 0.0, t, 1.0, [0.0, 0.0])
        return (K_AFFINE, *_grid_theta(matrix, H, W))
    if name == "Brightness":
        return (K_BRIGHTNESS, _f32(1.0 + mag))
    if name in ("Color", "Contrast"):
        ratio = 1.0 + mag
        return (K_COLOR if name == "Color" else K_CONTRAST, _f32(ratio), _f32(1.0 - ratio))
    if name == "Sharpness":
        return (K_SHARPNESS, _f32(1.0 - (1.0 + mag)))
    if name == "Posterize":
        bits = int(mag)
        return (K_POSTERIZE, float(0xFF if bits >= 8 else ((1 << bits) - 1) << (8 - bits)))
    if name == "Solarize":
        return (K_SOLARIZE, _f32(255.0 * mag))
    if name == "AutoContrast":
        return (K_AUTOCONTRAST,)
    if name == "Equalize":
        return (K_EQUALIZE,)
    if name == "Invert":
        return (K_INVERT,)
    return (K_IDENTITY,)


@functools.lru_cache(maxsize=64)
def chain_table(policy: str, H: int, W: int) -> np.ndarray:
    """Every outcome of one AutoAugment draw on an ``H x W`` image, encoded once: ``[25 * 16, AUG_CHAIN_PRM]`` float32, row
    ``16 * sub_policy + 4 * applied + signs`` (bit 0 of ``applied`` / ``signs``: the first entry is applied / negated,
    bit 1: the second).  A skipped entry is Identity; an applied first entry is op A, and a second entry applied alone is
    op B after an Identity op A."""
    names = chain_names()
    subs = sub_policies(policy)
    rows = np.zeros((len(subs) * 16, AUG_CHAIN_PRM), dtype=np.float32)
    rows[:, 12] = rows[:, COL_B + 7] = names.index("Identity")
    for i, sub in enumerate(subs):
        for applied in range(4):
            for signs in range(4):
                r = rows[16 * i + 4 * applied + signs]
                for k, (name, _, idx) in enumerate(sub):
                    if not applied >> k & 1:
                        continue
                    mag = aa_magnitude(policy, name, idx, bool(signs >> k & 1), H, W)
                    col = 0 if k == 0 else COL_B
                    code = op_code(name, mag, H, W)
                    r[col:col + len(code)] = code
                    ref = 12 if k == 0 else COL_B + 7
                    r[ref], r[ref + 1] = names.index(name), mag
    return rows


def erase_params(rng: np.random.Generator, H: int, W: int):
    """torchvision's ``RandomErasing.make_params``: up to 10 tries of area, log-ratio, ``h`` / ``w`` by ``round(sqrt)``,
    then ``i`` and ``j``; ``None`` when no try fits (the sample is left as it is)."""
    area = H * W
    lo, hi = math.log(ERASE_RATIO[0]), math.log(ERASE_RATIO[1])
    for _ in range(10):
        erase_area = area * rng.uniform(ERASE_SCALE[0], ERASE_SCALE[1])
        aspect = math.exp(rng.uniform(lo, hi))
        h = int(round(math.sqrt(erase_area * aspect)))
        w = int(round(math.sqrt(erase_area / aspect)))
        if not (h < H and w < W):
            continue
        i = int(rng.integers(0, H - h + 1))
        j = int(rng.integers(0, W - w + 1))
        return i, j, h, w
    return None


class BatchAugment:
    """The training-time input policy: per-sample TrivialAugment Wide or AutoAugment and random erasing draws, and their
    application.

    ``draw(n, H, W)`` runs on the host for every training batch and fills one of two pinned ``[n, width]`` tables
    (``width``: ``AUG_CHAIN_PRM`` for an AutoAugment policy, ``AUG_PRM`` otherwise; the
    prefetcher copies a batch while it stages the next one, so a table is not rewritten while its copy may be in flight).
    The draws come from ``numpy.random.Generator(PCG64([seed, rank, epoch, STREAM_ID]))``: ``set_epoch`` re-keys the stream,
    so a resume at an epoch boundary replays the same draws.  Without a seed, the seed comes from OS entropy.
    """

    def __init__(self, auto_augment: Optional[str] = "ta_wide", random_erase: float = 0.0, seed: Optional[int] = None,
                 rank: int = 0):
        if auto_augment not in (None, "ta_wide") + AUTOAUGMENT_POLICIES:
            raise ValueError("unknown auto-augment policy %r (one of 'ta_wide', %s)"
                             % (auto_augment, ", ".join(repr(p) for p in AUTOAUGMENT_POLICIES)))
        if not 0.0 <= random_erase <= 1.0:
            raise ValueError("random_erase must lie in [0, 1], got %r" % (random_erase,))
        self.auto_augment = auto_augment
        self.width = AUG_CHAIN_PRM if auto_augment in AUTOAUGMENT_POLICIES else AUG_PRM
        self.random_erase = float(random_erase)
        self.seed = (int(seed) if seed is not None else np.random.SeedSequence().entropy) % (1 << 128)
        self.rank = int(rank)
        pin = torch.cuda.is_available()
        self._slots = [torch.zeros((0, self.width), dtype=torch.float32) for _ in range(2)]
        self._events = [None, None]
        self._pin = pin
        self._next = 0
        self.set_epoch(0)

    def set_epoch(self, epoch: int) -> None:
        self.rng = np.random.Generator(np.random.PCG64([self.seed, self.rank, int(epoch), STREAM_ID]))

    def draw(self, n: int, H: int, W: int) -> torch.Tensor:
        """Draw the ops, magnitudes and erase boxes of the next ``n`` samples of ``H x W``; returns the (pinned) table."""
        n, H, W = int(n), int(H), int(W)
        if H * W > AUG_MAX_PIXELS:
            raise ValueError("augmentation of %dx%d images: more than %d pixels, beyond which Contrast's float32 mean is no "
                             "longer exact in torchvision's order" % (H, W, AUG_MAX_PIXELS))
        k = self._next
        self._next ^= 1
        if self._events[k] is not None:              # the copy of the batch before last still reads this slot
            self._events[k].synchronize()
            self._events[k] = None
        if self._slots[k].size(0) < n:
            t = torch.zeros((n, self.width), dtype=torch.float32)
            self._slots[k] = t.pin_memory() if self._pin else t
        tab = self._slots[k][:n]
        rng = self.rng
        if self.auto_augment in AUTOAUGMENT_POLICIES:
            rows = self._draw_chain(rng, n, H, W)
        else:
            rows = self._draw_trivial(rng, n, H, W)
        erase = rng.random(n) < self.random_erase if self.random_erase > 0 else np.zeros(n, dtype=bool)
        for s in np.flatnonzero(erase):
            box = erase_params(rng, H, W)
            if box is not None:
                rows[s, 7] = 1.0
                rows[s, 8:12] = box
        tab.copy_(torch.from_numpy(rows))
        return tab

    def _draw_trivial(self, rng, n: int, H: int, W: int) -> np.ndarray:
        """TrivialAugment Wide (or, without a policy, Identity) rows: op, bin and sign per sample."""
        n_ops = len(op_names())
        if self.auto_augment is not None:
            ops = rng.integers(0, n_ops, n)
            bins = rng.integers(0, NUM_BINS, n)
            neg = rng.random(n) < 0.5
        else:
            ops = bins = np.zeros(n, dtype=np.int64)
            neg = np.zeros(n, dtype=bool)
        rows = np.zeros((n, AUG_PRM), dtype=np.float32)
        names = op_names()
        for s in range(n):
            if self.auto_augment is not None:
                code = encode(int(ops[s]), int(bins[s]), bool(neg[s]), H, W)
                rows[s, :len(code)] = code
                rows[s, 12] = ops[s]
                rows[s, 13] = magnitude(int(ops[s]), int(bins[s]), bool(neg[s]), H, W)
            else:
                rows[s, 12] = names.index("Identity")
        return rows

    def _draw_chain(self, rng, n: int, H: int, W: int) -> np.ndarray:
        """AutoAugment rows: a sub-policy uniformly, each entry applied iff ``u <= p``, a signed magnitude negated iff
        ``v <= 0.5``; gathered from :func:`chain_table`."""
        subs = sub_policies(self.auto_augment)
        p = np.array([[e[1] for e in sub] for sub in subs], dtype=np.float64)
        sub = rng.integers(0, len(subs), n)
        applied = rng.random((n, 2)) <= p[sub]
        neg = rng.random((n, 2)) <= 0.5
        idx = 16 * sub + 4 * (applied[:, 0] + 2 * applied[:, 1]) + (neg[:, 0] + 2 * neg[:, 1])
        return chain_table(self.auto_augment, H, W)[idx]

    def copied(self, table: torch.Tensor, event) -> None:
        """The consumer enqueued its copy of ``table`` (the last ``draw``); ``event`` completes when it is done."""
        self._events[self._next ^ 1] = event

    @staticmethod
    def apply(src: torch.Tensor, prm: torch.Tensor, a: torch.Tensor, b: torch.Tensor, dtype: torch.dtype,
              channels_last: bool) -> torch.Tensor:
        """Augment, normalise (``x * a[c] + b[c]``) and erase the uint8 ``[n, 3, H, W]`` batch ``src``: the GPU kernel, or
        :meth:`reference_apply` on CPU tensors."""
        if not src.is_cuda:
            return BatchAugment.reference_apply(src, prm, a, b, dtype, channels_last)
        from .. import _ext
        code = {torch.float32: 0, torch.bfloat16: 1, torch.float16: 2}[dtype]
        _ext.note_launch()
        return _ext.lib().augment_normalize(src, prm, a, b, code, channels_last)

    @staticmethod
    def reference_apply(src: torch.Tensor, prm: torch.Tensor, a: torch.Tensor, b: torch.Tensor, dtype: torch.dtype,
                        channels_last: bool) -> torch.Tensor:
        """The CPU path: ``transforms.v2.functional`` per sample (through torchvision's own op dispatch; op B of a two-op row
        on op A's output), the normalisation ``fp32(x * a[c] + b[c])`` rounded once, as the kernels' FMA, and the erase box
        set to 0."""
        pol = _policy()
        names = chain_names()
        p = prm.detach().cpu().numpy()
        a64 = a.detach().cpu().double().view(1, 3, 1, 1)
        b64 = b.detach().cpu().double().view(1, 3, 1, 1)
        src = src.cpu()
        out = []
        for s in range(src.size(0)):
            img = src[s]
            for col in ((12, COL_B + 7) if p.shape[1] == AUG_CHAIN_PRM else (12,)):
                img = pol._apply_image_or_video_transform(img, names[int(p[s, col])], float(p[s, col + 1]),
                                                          interpolation=pol.interpolation, fill=pol._fill)
            out.append(img)
        x = torch.stack(out).double()
        # x * a + b is exact in float64 (8-bit x times a 24-bit a, plus b, spans fewer than 53 bits): one rounding to fp32
        y = (x * a64 + b64).float()
        for s in range(src.size(0)):
            if p[s, 7] != 0:
                i, j, h, w = (int(v) for v in p[s, 8:12])
                y[s, :, i:i + h, j:j + w] = 0.0
        y = y.to(dtype)
        return y.contiguous(memory_format=torch.channels_last) if channels_last else y
