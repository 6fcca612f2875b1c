"""Mixed-precision modulated deformable convolution without a GPU: the 16-bit C entry points and their argument
checks, the dtype rule as a pure function, the column chunk size by element size, and the pre-training harness's
`backbone_autocast` option."""
import ctypes
import re

import pytest
import torch

from vidar_b200 import _lib

F32, F16, BF16, F64 = torch.float32, torch.float16, torch.bfloat16, torch.float64


def test_half_entry_points_report_bad_arguments():
    """Validated before any launch: every call returns VIDAR_E_INVALID with a message (a dummy non-null address
    stands in for device memory; nothing is touched)."""
    L = _lib.lib()
    N, X = None, ctypes.c_void_p(0x1000)
    geom = [2, 16, 10, 12, 10, 12, 3, 3, 1, 1, 1, 1, 1, 1]        # N C H W Ho Wo kh kw sh sw ph pw dh dw

    def g(**k):
        names = ["N", "C", "H", "W", "Ho", "Wo", "kh", "kw", "sh", "sw", "ph", "pw", "dh", "dw", "n0", "nb"]
        vals = dict(zip(names, geom + [0, 2]))
        vals.update(k)
        return [vals[n] for n in names]

    im2col, col2im = L.vidar_dcn_im2col_half, L.vidar_dcn_col2im_half
    cases = []
    for code in (1, 2):
        cases += [
            (im2col, (N, X, X, X, code, *g(), N), b"null pointer"),
            (im2col, (X, X, X, X, code, *g(C=0), N), b"bad sizes"),
            (im2col, (X, X, X, X, code, *g(Ho=9), N), b"does not match the convolution"),
            (im2col, (X, X, X, X, code, *g(n0=1, nb=2), N), b"bad image range"),
            (col2im, (X, X, X, X, X, X, N, code, *g(), N), b"null pointer"),
            (col2im, (X, X, X, X, X, X, X, code, *g(dw=2), N), b"does not match the convolution"),
            (col2im, (X, X, X, X, X, X, X, code, *g(n0=3, nb=0), N), b"bad image range"),
        ]
    for code in (0, 3, -1):
        cases += [(im2col, (X, X, X, X, code, *g(), N), b"unsupported dtype"),
                  (col2im, (X, X, X, X, X, X, X, code, *g(), N), b"unsupported dtype")]
    for fn, args, needle in cases:
        rc = fn(*args)
        assert rc == 1, (fn.__name__, args, rc, L.vidar_last_error())
        assert needle in L.vidar_last_error(), (fn.__name__, L.vidar_last_error())
    for code in (1, 2):          # an empty image range is a no-op
        assert im2col(X, X, X, X, code, *g(nb=0), N) == 0
        assert col2im(X, X, X, X, X, X, X, code, *g(n0=2, nb=0), N) == 0


def test_dtype_codes_match_the_header():
    from vidar_b200.dcn import HALF_DTYPE_CODES
    with open(_lib.HEADER) as fh:
        src = fh.read()
    codes = {name: int(v) for name, v in re.findall(r"#define VIDAR_DTYPE_(\w+) (\d+)", src)}
    assert codes == {"F16": HALF_DTYPE_CODES[F16], "BF16": HALF_DTYPE_CODES[BF16]}


@pytest.mark.parametrize("dts, want", [
    ((F32, F32, F32, F32, F32), F32),
    ((F32, F32, F32, F32, None), F32),
    ((F16, F16, F16, F16, F16), F16),
    ((BF16, BF16, BF16, BF16, None), BF16),
    ((F32, F16, F32, F32, F32), F16),          # fp32 input, fp16 offset: fp16
    ((F16, F32, F16, F16, F16), F32),          # fp16 input, fp32 offset: the fp32 path
    ((F16, BF16, F32, F32, None), BF16),       # an fp32 weight under bf16 autocast
    ((F32, BF16, F16, F32, F16), BF16),
])
def test_compute_dtype_is_the_offset_dtype(dts, want):
    from vidar_b200.dcn import compute_dtype
    assert compute_dtype(*dts) is want


@pytest.mark.parametrize("dts", [
    (F32, F64, F32, F32, None),
    (F64, F32, F32, F32, None),
    (F16, F16, F64, F16, None),
    (F32, F32, F32, F64, None),
    (F32, F32, F32, F32, F64),
    (F32, torch.int32, F32, F32, None),
])
def test_compute_dtype_rejects_other_dtypes(dts):
    from vidar_b200.dcn import compute_dtype
    with pytest.raises(TypeError, match="float32"):
        compute_dtype(*dts)


def test_chunk_counts_bytes_by_element_size():
    from vidar_b200 import dcn
    per_image = 58 * 100 * 9 * 256
    fp32 = dcn.chunk_images(64, per_image)
    assert fp32 == dcn.MAX_COLS_BYTES // (4 * per_image) and dcn.chunk_images(64, per_image, 2) == 2 * fp32
    assert dcn.chunk_images(6, dcn.MAX_COLS_BYTES // 2, 2) == 1


def test_backbone_autocast_keeps_the_state_dict():
    """The option holds no state: SyntheticViDAR(backbone_autocast=...) has the default model's pinned keys."""
    import hashlib

    from tests.test_dcn_cpu import SYNTHETIC_VIDAR_KEYS_SHA256
    from vidar_b200.pretrain import SyntheticViDAR
    for dt in (None, F16, BF16):
        m = SyntheticViDAR(backbone_autocast=dt)
        assert m.backbone_autocast is dt
        lines = "\n".join(f"{k} {tuple(v.shape)}" for k, v in sorted(m.state_dict().items()))
        assert hashlib.sha256(lines.encode()).hexdigest() == SYNTHETIC_VIDAR_KEYS_SHA256
    with pytest.raises(ValueError, match="backbone_autocast"):
        SyntheticViDAR(encoder_layers=1, decoder_layers=1, backbone_autocast=F32)
