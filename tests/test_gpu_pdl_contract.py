"""The PDL contract, kernel by kernel: before pdl_wait() a kernel reads nothing an earlier kernel of the step writes, and
writes nothing to global memory (csrc/ptx.cuh).

A kernel that breaks it still gets the right bits whenever its predecessor happens to finish first, which it usually
does, so comparing PDL on with PDL off (test_gpu_ordering.py) cannot see the race.  Here the predecessor is made late on
purpose: vlo_op_pdl_arm arms a probe kernel that each entry launches right before its first PDL launch.  The probe lets
the kernel under test launch at once, spins on the global timer for SPIN_NS while that kernel's CTAs become resident on
the other SMs, and only then
  * late write: copies an operand's real values over a poisoned copy (NaN, or a different finite pattern where NaN is
    not a value of the type or could stall the kernel).  A kernel that read the operand before its wait computes from
    the poison;
  * late read: snapshots an output or workspace region (an exchange: the region gets back the values the kernel must
    find there).  A kernel that wrote there before its wait shows in the snapshot.
Every output of a case must equal, bit for bit, a serial run of the entry on the real values, and every snapshot must
equal the region's contents before the launch.  Each case is one probe and one launch, and asserts that its probe ran,
so an entry without the hook cannot pass vacuously.

What counts as a predecessor's data.  Late operands are those another kernel of the step produces: activations, their
token scales, stream-K planes, the residual stream, q and the K/V rows a step appends, logits, frames and camera
planes.  Weights, scales of weights, RoPE tables, tables uploaded by memcpy and K/V rows of earlier steps are allowed
before the wait and are never written late; in particular the attention cases late-write only the rows of the current
step, including those that share the last 64-key block with cached rows.

Coverage.  attn_merge_kernel follows the attention kernel inside attn_run, so the probe reaches it only through the
attention kernel's own wait (its output region is checked all the same).  Kernels launched with <<<>>> (the embedding
gathers, probe_attn, pool, the CLS residual, the KV-cache kernels, fp16-input LayerNorm) are serialised by the stream
and out of scope.

The controls come first: a canary launched through the product's launch helper must be caught reading before its wait
under a late write and writing before its wait under a late read, so a device or driver that stops overlapping grids
fails this file instead of turning it into a no-op."""
import ctypes as C
import math
import os

import pytest
import torch

pytestmark = pytest.mark.gpu

if os.environ.get("VLO_NO_PDL") == "1":
    pytest.skip("PDL is off in this process (VLO_NO_PDL=1): no kernel can start before its predecessor ends",
                allow_module_level=True)

# How long the probe holds back the operand.  The dependents of a launch become resident within microseconds; 200 us
# leaves room for every CTA of a full-SM persistent grid to reach its wait.
SPIN_NS = 200_000
FMT_F16, FMT_BF16, FMT_E4M3, FMT_E4M3_A8, FMT_I4 = 0, 1, 2, 3, 4
EPI_STORE16 = 1
FIX_MAX_PLANES = 8
PAD_WS = 3                    # extra rows behind outputs, so a write past the end shows as a difference too


@pytest.fixture(scope="module")
def lib():
    from videollm_online_b200 import _lib
    return _lib.load()


def _p(t):
    return None if t is None else C.c_void_p(t.data_ptr())


def _st():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _check(rc, what):
    from videollm_online_b200._lib import check
    check(rc, what)


def _bytes(t):
    return t.contiguous().view(torch.uint8).flatten()


def _same_bits(a, b):
    return a.dtype == b.dtype and a.shape == b.shape and torch.equal(_bytes(a), _bytes(b))


def _n_sm():
    return torch.cuda.get_device_properties(0).multi_processor_count


# ================================================================================================ case machinery
class Region:
    """n_chunks chunks of `elems` elements of tensor `name`, chunk i starting at element first + i * stride.
    poison: the late-write fill (None: NaN for float types, 0x7F - an e4m3 NaN - for uint8).  marker: what a late-read
    region holds at the launch instead of its values (the probe's exchange puts them back), for regions the kernel
    reads after its wait and whose values an early write would not change (zero counters)."""

    def __init__(self, name, first=0, elems=None, n_chunks=1, stride=0, poison=None, marker=None):
        self.name, self.first, self.elems, self.n_chunks, self.stride = name, first, elems, n_chunks, stride
        self.poison, self.marker = poison, marker

    def chunks(self, t):
        n = t.numel() - self.first if self.elems is None else self.elems() if callable(self.elems) else self.elems
        return [(self.first + i * self.stride, n) for i in range(self.n_chunks)]

    def arm_args(self, t, other):
        """(dst, src, bytes, n_chunks, chunk_stride) of this region of t, paired with the same region of `other`"""
        es = t.element_size()
        (e0, n), = self.chunks(t)[:1]
        return (C.c_void_p(t.data_ptr() + e0 * es), C.c_void_p(other.data_ptr() + e0 * es), n * es, self.n_chunks,
                self.stride * es)

    def gather(self, t):
        flat = t.view(-1)
        return torch.cat([_bytes(flat[a:a + n]) for a, n in self.chunks(t)])

    def fill(self, t, v=None):
        flat = t.view(-1)
        if v is None:
            v = self.poison
        if v is None:
            v = float("nan") if t.dtype.is_floating_point else 0x7F
        for a, n in self.chunks(t):
            flat[a:a + n].fill_(v)


class Case:
    """make() -> dict of fresh device tensors (the same values on every call); call(lib, s) runs the entry once.
    outs: the tensors whose bits must equal the serial run; late_in / late_out: the regions of the two kinds of case."""

    def __init__(self, name, make, call, outs, late_in, late_out):
        self.name, self.make, self.call, self.outs = name, make, call, outs
        self.late_in = {r.name if isinstance(r, Region) else r: (r if isinstance(r, Region) else Region(r)) for r in late_in}
        self.late_out = {r.name if isinstance(r, Region) else r: (r if isinstance(r, Region) else Region(r))
                         for r in late_out}


_WEIGHTS = {}


def _weight(key, fn):
    """operands no kernel writes, built once per module run"""
    if key not in _WEIGHTS:
        _WEIGHTS[key] = fn()
    return _WEIGHTS[key]


def _gen(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


def _nan(*shape, dtype=torch.bfloat16):
    return torch.full(shape, float("nan"), dtype=dtype, device="cuda")


# ================================================================================================ GEMM operands
def _w16(N, K, dtype=torch.bfloat16):
    return _weight(("w16", N, K, dtype), lambda: (torch.randn(N, K, device="cuda", generator=_gen(N + K)) /
                                                  math.sqrt(K)).to(dtype))


def _wq(fmt, N, K):
    """(codes, scale) of the bf16 weight: e4m3 codes + fp32 row scales, or packed int4 codes + bf16 group scales"""
    from videollm_online_b200 import weights as W
    if fmt in (FMT_E4M3, FMT_E4M3_A8):
        return _weight(("f8", N, K), lambda: W.quantize_fp8_rows(_w16(N, K)))
    def i4():
        q, s = W.quantize_int4_groups(_w16(N, K))
        return W.pack_int4_codes(q), s
    return _weight(("i4", N, K), i4)


def _x(T, K, seed, dtype=torch.bfloat16):
    return torch.randn(T, K, device="cuda", generator=_gen(seed)).to(dtype)


def _x8(T, K, seed):
    """e4m3 activation codes [T, K] and fp32 token scales [T]"""
    from videollm_online_b200 import weights as W
    return W.quantize_fp8_rows(_x(T, K, seed))


def _planes_of(lib, fmt, mode, w, N, x, T, K):
    """the plane count a gemm_ws launch of these operands needs (its planning query)"""
    plan = (C.c_int32 * 3)()
    _check(lib.vlo_op_gemm_ws_tiled(fmt, mode, _p(w), N, _p(x), T, K, None, N, T * N, None, 0, 0, 0, 0, plan, _st()),
           "gemm_ws plan")
    return plan[2]


DEC_SHAPES = {"8b": (4096, 4096, 11), "tiny": (256, 256, 5)}       # (N, K, T): o_proj of Llama-3-8B, one token tile
SWIGLU_SHAPES = {"8b": (28672, 4096, 11), "tiny": (256, 256, 5)}   # gate|up of Llama-3-8B
PREFILL_SHAPES = {"8b": (4096, 4096, 300), "tiny": (256, 256, 129)}
VIT_SHAPES = {"siglip": (1152, 1152, 729 * 2), "tiny": (128, 128, 100)}


def _gemm_ws_case(fmt, mode, shape):
    N, K, T = DEC_SHAPES[shape]
    dt = torch.float16 if fmt == FMT_F16 else torch.bfloat16

    def make(lib):
        w, x = _w16(N, K, dt), _x(T, K, 1, dt)
        if mode == 0:
            out = _nan(_planes_of(lib, fmt, 0, w, N, x, T, K) * T * N + PAD_WS, dtype=torch.float32)
        else:
            out = _nan(T + PAD_WS, N, dtype=dt)
        return dict(w=w, x=x, out=out)

    def call(lib, s):
        _check(lib.vlo_op_gemm_ws_tiled(fmt, mode, _p(s["w"]), N, _p(s["x"]), T, K, _p(s["out"]), N, T * N, None, 0, 0, 0,
                                        0, None, _st()), "gemm_ws_tiled")
    name = f"gemm_ws_tiled/{'fp16' if fmt == FMT_F16 else 'bf16'}/mode{mode}/{shape}"
    return Case(name, make, call, ["out"], ["x"], ["out"])


def _gemm_ws_q_case(fmt, shape):
    """gemm_ws_f8 / gemm_ws_a8 / gemm_ws_i4: stream-K partial planes"""
    N, K, T = DEC_SHAPES[shape]
    entry = {FMT_E4M3: "f8", FMT_E4M3_A8: "a8", FMT_I4: "i4"}[fmt]

    def make(lib):
        w, sc = _wq(fmt, N, K)
        s = dict(w=w, sc=sc)
        if fmt == FMT_E4M3_A8:
            s["x"], s["xs"] = _x8(T, K, 2)
        else:
            s["x"] = _x(T, K, 2)
        planes = C.c_int(0)
        fn = getattr(lib, f"vlo_op_gemm_ws_{entry}")
        args = [_p(w), _p(sc), N, _p(s["x"])] + ([_p(s["xs"])] if fmt == FMT_E4M3_A8 else []) + [T, K]
        _check(fn(*args, None, T * N, 0, C.byref(planes), _st()), "plan")
        s["out"] = _nan(planes.value * T * N + PAD_WS, dtype=torch.float32)
        return s

    def call(lib, s):
        fn = getattr(lib, f"vlo_op_gemm_ws_{entry}")
        args = [_p(s["w"]), _p(s["sc"]), N, _p(s["x"])] + ([_p(s["xs"])] if fmt == FMT_E4M3_A8 else []) + [T, K]
        _check(fn(*args, _p(s["out"]), T * N, 0, None, _st()), f"gemm_ws_{entry}")
    late_in = ["x", "xs"] if fmt == FMT_E4M3_A8 else ["x"]
    return Case(f"gemm_ws_{entry}/{shape}", make, call, ["out"], late_in, ["out"])


def _tiles_q_case(fmt, shape):
    N, K, T = DEC_SHAPES[shape]

    def make(lib):
        w, sc = _wq(fmt, N, K)
        return dict(w=w, sc=sc, x=_x(T, K, 3), out=_nan(T + PAD_WS, N))

    def call(lib, s):
        _check(lib.vlo_op_gemm_ws_tiles_q(fmt, _p(s["w"]), _p(s["sc"]), N, _p(s["x"]), T, K, _p(s["out"]), N, 0, None,
                                          _st()), "gemm_ws_tiles_q")
    return Case(f"gemm_ws_tiles_q/{'e4m3' if fmt == FMT_E4M3 else 'int4'}/{shape}", make, call, ["out"], ["x"], ["out"])


def _swiglu_case(fmt, shape):
    N, K, T = SWIGLU_SHAPES[shape]
    entry = {FMT_BF16: "", FMT_E4M3: "_f8", FMT_E4M3_A8: "_a8", FMT_I4: "_i4"}[fmt]

    def make(lib):
        s = {}
        if fmt == FMT_BF16:
            s["w"] = _w16(N, K)
        else:
            s["w"], s["sc"] = _wq(fmt, N, K)
        if fmt == FMT_E4M3_A8:
            s["x"], s["xs"] = _x8(T, K, 4)
        else:
            s["x"] = _x(T, K, 4)
        s["act"] = _nan(T + PAD_WS, N // 2)
        s["planes"] = _nan(FIX_MAX_PLANES * T * N, dtype=torch.float32)
        s["flags"] = torch.zeros(N // 128 + PAD_WS, dtype=torch.int32, device="cuda")
        return s

    def call(lib, s):
        fn = getattr(lib, f"vlo_op_gemm_swiglu{entry}")
        head = [_p(s["w"])] + ([] if fmt == FMT_BF16 else [_p(s["sc"])]) + [N, _p(s["x"])]
        head += [_p(s["xs"])] if fmt == FMT_E4M3_A8 else []
        _check(fn(*head, T, K, _p(s["act"]), _p(s["planes"]), s["planes"].numel(), _p(s["flags"]), s["flags"].numel(),
                  _st()), f"gemm_swiglu{entry}")
    late_in = ["x", "xs"] if fmt == FMT_E4M3_A8 else ["x"]
    # the finisher resets each counter after its wait: one reset before it would race with a previous launch's arrivals
    flags = Region("flags", marker=0x5A5A5A5A)
    return Case(f"gemm_swiglu{entry}/{shape}", make, call, ["act", "flags"], late_in, ["act", "planes", flags])


def _prefill_case(form, shape):
    N, K, T = PREFILL_SHAPES[shape]
    fmt = {"bf16": FMT_BF16, "fp8": FMT_E4M3, "w8a8": FMT_E4M3_A8, "int4": FMT_I4}[form]

    def make(lib):
        s = {}
        if fmt == FMT_BF16:
            s["w"] = _w16(N, K)
        else:
            s["w"], s["sc"] = _wq(fmt, N, K)
        if fmt == FMT_E4M3_A8:
            s["x"], s["xs"] = _x8(T, K, 5)
        else:
            s["x"] = _x(T, K, 5)
        s["out"] = _nan(T + PAD_WS, N, dtype=torch.float32)
        return s

    def call(lib, s):
        if fmt == FMT_BF16:
            _check(lib.vlo_op_gemm_prefill(0, _p(s["w"]), N, _p(s["x"]), T, K, 0, _p(s["out"]), _st()), "gemm_prefill")
            return
        sc = s["sc"] if fmt in (FMT_E4M3, FMT_E4M3_A8) else None
        gs = s["sc"] if fmt == FMT_I4 else None
        _check(lib.vlo_op_gemm_prefill_q(fmt, 0, _p(s["w"]), _p(sc), _p(gs), N, _p(s["x"]), _p(s.get("xs")), T, K, 0,
                                         _p(s["out"]), _st()), "gemm_prefill_q")
    late_in = ["x", "xs"] if fmt == FMT_E4M3_A8 else ["x"]
    name = "gemm_prefill" if fmt == FMT_BF16 else f"gemm_prefill_q/{form}"
    return Case(f"{name}/{shape}", make, call, ["out"], late_in, ["out"])


def _vit_gemm_case(entry, shape):
    N, K, M = VIT_SHAPES[shape]

    def make(lib):
        bias = _weight(("bias", N), lambda: torch.randn(N, device="cuda", generator=_gen(N)))
        return dict(w=_w16(N, K, torch.float16), bias=bias, x=_x(M, K, 6, torch.float16),
                    out=_nan(M + PAD_WS, N, dtype=torch.float16))

    def call(lib, s):
        if entry == "gemm_vit":
            _check(lib.vlo_op_gemm_vit(_p(s["w"]), N, _p(s["x"]), M, K, _p(s["out"]), N, _p(s["bias"]), 0, 0, _st()),
                   "gemm_vit")
        else:
            _check(lib.vlo_op_gemm(EPI_STORE16, 0, _p(s["x"]), M, _p(s["w"]), N, K, _p(s["out"]), N, _p(s["bias"]), None,
                                   0, 128, _st()), "gemm")
    return Case(f"{entry}/{shape}", make, call, ["out"], ["x"], ["out"])


# ================================================================================================ decoder kernels
def _resid_case(q8, shape):
    H, T, k = {"8b": (4096, 11, 4096), "tiny": (256, 3, 256)}[shape]

    def make(lib):
        g = _gen(H + T)
        s = dict(part=torch.randn(FIX_MAX_PLANES, T, H, device="cuda", generator=g),
                 h=torch.randn(T, H, device="cuda", generator=g).bfloat16(),
                 w=_weight(("norm", H), lambda: (1 + 0.25 * torch.randn(H, device="cuda", generator=_gen(H))).bfloat16()),
                 xn=_nan(T + PAD_WS, H), xn_last=_nan(2, H),
                 li=torch.tensor([-1] * (T - 1) + [0], dtype=torch.int32, device="cuda"))
        if q8:
            s["xq"] = torch.full((T + PAD_WS, H), 0x7F, dtype=torch.uint8, device="cuda")
            s["xs"] = _nan(T + PAD_WS, dtype=torch.float32)
        return s

    def call(lib, s):
        if q8:
            _check(lib.vlo_op_resid_rmsnorm_q8(_p(s["part"]), k, 0, _p(s["h"]), _p(s["w"]), _p(s["xn"]), _p(s["xn_last"]),
                                               _p(s["li"]), _p(s["xq"]), _p(s["xs"]), T, H, 1e-5, _st()),
                   "resid_rmsnorm_q8")
        else:
            _check(lib.vlo_op_resid_rmsnorm(_p(s["part"]), k, 0, _p(s["h"]), _p(s["w"]), _p(s["xn"]), _p(s["xn_last"]),
                                            _p(s["li"]), T, H, 1e-5, _st()), "resid_rmsnorm")
    outs = ["h", "xn", "xn_last"] + (["xq", "xs"] if q8 else [])
    return Case(f"resid_rmsnorm{'_q8' if q8 else ''}/{shape}", make, call, outs, ["part", "h"], outs)


def _quant_rows_case():
    T, K = 11, 14336

    def make(lib):
        return dict(x=_x(T, K, 7), q=torch.full((T + PAD_WS, K), 0x7F, dtype=torch.uint8, device="cuda"),
                    s=_nan(T + PAD_WS, dtype=torch.float32))

    def call(lib, s):
        _check(lib.vlo_op_quant_rows_e4m3(_p(s["x"]), T, K, _p(s["q"]), _p(s["s"]), _st()), "quant_rows_e4m3")
    return Case("quant_rows_e4m3/8b", make, call, ["q", "s"], ["x"], ["q", "s"])


ROPE_POS = 13100


def _rope():
    from videollm_online_b200 import tiny_config, weights as W
    return _weight(("rope",), lambda: W.rope_tables(tiny_config(), ROPE_POS, "cuda"))


def _qkv_rope_case():
    """the 8B model's q|k|v fix-up for 11 tokens at positions 12990 .. 13000 of a contiguous cache: the appended rows
    of each kv head are one chunk"""
    nh, nkv, T, k, ld, p0 = 32, 8, 11, 4096, ROPE_POS, 12990
    width = (nh + 2 * nkv) * 128

    def make(lib):
        return dict(part=torch.randn(FIX_MAX_PLANES, T, width, device="cuda", generator=_gen(width)),
                    q=_nan(T + PAD_WS, nh, 128), kc=_nan(nkv * ld, 128), vc=_nan(nkv * ld, 128))

    def call(lib, s):
        cos, sin = _rope()
        pos = (C.c_int32 * T)(*range(p0, p0 + T))
        rows = (C.c_int64 * T)(*range(p0, p0 + T))
        _check(lib.vlo_op_qkv_rope_append(_p(s["part"]), k, 0, _p(cos), _p(sin), ROPE_POS, pos, rows, ld, _p(s["q"]),
                                          _p(s["kc"]), _p(s["vc"]), T, nh, nkv, _st()), "qkv_rope_append")
    rows = [Region(n, first=p0 * 128, elems=T * 128, n_chunks=nkv, stride=ld * 128) for n in ("kc", "vc")]
    return Case("qkv_rope_append/8b", make, call, ["q", "kc", "vc"], ["part"], ["q"] + rows)


# ================================================================================================ attention
HQ, HK, D = 32, 8, 128


def _attn_ws_prefix(n_tok):
    """bytes of ws_o and ws_ml at the head of an attention workspace (attn.cu: attn_ws_bytes, one sequence)"""
    G = HQ // HK
    per = max(1, 64 // G)
    chunks = n_tok // per + 2
    slots = (_n_sm() + HK * chunks) * 128 + (_n_sm() + HK) * G * n_tok
    a256 = lambda b: (b + 255) // 256 * 256
    return a256(slots * D * 4) + a256(slots * 2 * 4)


def _attn_case(kind, kv_len, segs=None):
    """kind "contiguous": vlo_op_attn_kvappend over [HK][kv_len + 7][128]; "paged" / "segments": a pool whose pages
    the table scatters.  The step's n_tok rows are the last ones; the earlier rows are cached (allowed before the
    wait), so only the new rows are late-written, per kv head."""
    n_tok = sum(segs) if segs else 11
    blocks = (kv_len + 63) // 64

    def kv_pool(g):
        return (torch.randn(n_pages * HK * 64, D, device="cuda", generator=g) * 2).bfloat16()
    n_pages = blocks + 3
    table = [n_pages - 1 - b for b in range(blocks)]       # blocks in reverse page order, three pages unused

    def make(lib):
        g = _gen(kv_len * 3 + n_tok)
        s = dict(q=torch.randn(n_tok, HQ, D, device="cuda", generator=g).bfloat16(), out=_nan(n_tok + PAD_WS, HQ * D))
        if kind == "contiguous":
            s["k"] = (torch.randn(HK, kv_len + 7, D, device="cuda", generator=g) * 2).bfloat16()
            s["v"] = torch.randn(HK, kv_len + 7, D, device="cuda", generator=g).bfloat16()
        else:
            s["k"], s["v"] = kv_pool(g), kv_pool(g)
            s["pt"] = torch.tensor(table, dtype=torch.int32, device="cuda")
        if kind != "segments":
            s["ws"] = _nan(lib.vlo_op_attn_ws_bytes(n_tok, HQ, D, kv_len) // 4, dtype=torch.float32)
        return s

    def call(lib, s):
        if kind == "contiguous":
            _check(lib.vlo_op_attn_kvappend(_p(s["q"]), _p(s["k"]), _p(s["v"]), _p(s["out"]), _p(s["ws"]), n_tok, HQ, HK,
                                            D, kv_len, kv_len + 7, _st()), "attn_kvappend")
        elif kind == "paged":
            _check(lib.vlo_op_attn_kvappend_paged(_p(s["q"]), _p(s["k"]), _p(s["v"]), _p(s["pt"]), n_pages, _p(s["out"]),
                                                  _p(s["ws"]), n_tok, HQ, HK, D, kv_len, _st()), "attn_kvappend_paged")
        else:
            lens = (C.c_int32 * len(segs))(*segs)
            _check(lib.vlo_op_attn_kvappend_segments(_p(s["q"]), _p(s["k"]), _p(s["v"]), _p(s["pt"]), n_pages,
                                                     _p(s["out"]), len(segs), lens, HQ, HK, D, kv_len, _st()),
                   "attn_kvappend_segments")
    t0 = kv_len - n_tok
    if kind == "contiguous":
        new = [Region(n, first=t0 * D, elems=n_tok * D, n_chunks=HK, stride=(kv_len + 7) * D) for n in ("k", "v")]
    else:   # the new rows lie in the last block, beside cached rows of it: one chunk per kv head of its page
        assert t0 // 64 == blocks - 1 and t0 % 64 > 0
        page = table[blocks - 1]
        new = [Region(n, first=(page * HK * 64 + t0 % 64) * D, elems=n_tok * D, n_chunks=HK, stride=64 * D)
               for n in ("k", "v")]
    late_out = ["out"] + ([] if kind == "segments" else [Region("ws", elems=lambda: _attn_ws_prefix(n_tok) // 4)])
    plan = "plain" if not segs else "cluster" if segs[0] > 1 else "packed"
    case = Case(f"attn_kvappend_{kind}/{plan}/kv{kv_len}", make, call, ["out"], ["q"] + new, late_out)
    case.segs = segs
    return case


# ================================================================================================ logits
def _logits(n, V, seed):
    return (torch.randn(n, V, device="cuda", generator=_gen(seed)) * 3).bfloat16()


LOGITS_POISON = -3.0          # finite: every id equally likely, far from the real rows' argmax and probabilities


def _decision_case():
    n, V = 2, 128256

    def make(lib):
        return dict(logits=_logits(n, V, 8), out=torch.full((n + PAD_WS, 8), -7, dtype=torch.int32, device="cuda"))

    def call(lib, s):
        _check(lib.vlo_op_decision(_p(s["logits"]), n, V, 13, _p(s["out"]), _st()), "decision")
    return Case("decision/8b", make, call, ["out"], [Region("logits", poison=LOGITS_POISON)], ["out"])


def _sample_case():
    n, V = 2, 128256
    pen = [5, 17, 99]

    def make(lib):
        return dict(logits=_logits(n, V, 9), ids=torch.full((n + PAD_WS,), -7, dtype=torch.int32, device="cuda"),
                    info=torch.full((n + PAD_WS, 4), -7, dtype=torch.int32, device="cuda"))

    def call(lib, s):
        from videollm_online_b200._lib import VloSampleRow
        rows = (VloSampleRow * n)()
        for r, kw in zip(rows, [dict(seed=3, position=4, temperature=0.7, top_k=40, top_p=0.9, repetition_penalty=1.3,
                                     penalty_offset=0, penalty_count=len(pen)),
                                dict(seed=5, position=0, temperature=1.0, top_k=0, top_p=1.0, repetition_penalty=1.0)]):
            for k, v in kw.items():
                setattr(r, k, v)
        ids = (C.c_int32 * len(pen))(*pen)
        _check(lib.vlo_op_sample(_p(s["logits"]), n, V, rows, C.cast(ids, C.c_void_p), len(pen), _p(s["ids"]),
                                 _p(s["info"]), _st()), "sample")
    return Case("sample/8b", make, call, ["ids", "info"], [Region("logits", poison=LOGITS_POISON)], ["ids", "info"])


# ================================================================================================ vision tower
VB, VS, VPS, VC = 2, 384, 16, 1152         # frames, image size, patch size and SigLIP's width
VN = (VS // VPS) ** 2


def _patchify_case():
    def make(lib):
        f = torch.randint(0, 256, (VB, 3, VS, VS), dtype=torch.uint8, device="cuda", generator=_gen(10))
        return dict(frames=f, out=_nan(VB * VN + PAD_WS, 3 * VPS * VPS, dtype=torch.float16))

    def call(lib, s):
        _check(lib.vlo_op_patchify(_p(s["frames"]), VB, VS, VPS, _p(s["out"]), _st()), "patchify")
    return Case("patchify", make, call, ["out"], [Region("frames", poison=0x5A)], ["out"])


def _vit_ln_w():
    return _weight(("ln", VC), lambda: (1 + 0.1 * torch.randn(VC, device="cuda", generator=_gen(11)),
                                        0.02 * torch.randn(VC, device="cuda", generator=_gen(12))))


def _layernorm_case():
    rows = VB * VN

    def make(lib):
        return dict(x=torch.randn(rows, VC, device="cuda", generator=_gen(13)) * 4,
                    out16=_nan(rows + PAD_WS, VC, dtype=torch.float16), out32=_nan(rows + PAD_WS, VC, dtype=torch.float32))

    def call(lib, s):
        w, b = _vit_ln_w()
        _check(lib.vlo_op_vit_layernorm(_p(s["x"]), 0, rows, VC, _p(w), _p(b), _p(s["out16"]), _p(s["out32"]), 1e-6,
                                        _st()), "vit_layernorm")
    return Case("vit_layernorm/fp32", make, call, ["out16", "out32"], ["x"], ["out16", "out32"])


def _fix_ln_case():
    rows, k, bn = VB * VN, 4352, 128

    def make(lib):
        g = _gen(14)
        return dict(part=torch.randn(FIX_MAX_PLANES, rows, VC, device="cuda", generator=g),
                    h=torch.randn(rows, VC, device="cuda", generator=g) * 4,
                    out16=_nan(rows + PAD_WS, VC, dtype=torch.float16), out32=_nan(rows + PAD_WS, VC, dtype=torch.float32))

    def call(lib, s):
        w, b = _vit_ln_w()
        bias = _weight(("bias", VC), lambda: torch.randn(VC, device="cuda", generator=_gen(VC)))
        _check(lib.vlo_op_vit_fix_ln(_p(s["part"]), rows, VC, k, bn, 0, _p(bias), _p(s["h"]), _p(w), _p(b),
                                     _p(s["out16"]), _p(s["out32"]), 1e-6, _st()), "vit_fix_ln")
    return Case("vit_fix_ln", make, call, ["h", "out16", "out32"], ["part", "h"], ["h", "out16", "out32"])


def _vit_attn_case():
    def make(lib):
        return dict(qkv=(torch.randn(VB * VN, 3 * VC, device="cuda", generator=_gen(15)) * 2).half(),
                    out=_nan(VB * VN + PAD_WS, VC, dtype=torch.float16))

    def call(lib, s):
        _check(lib.vlo_op_vit_attn(_p(s["qkv"]), _p(s["out"]), VB, VN, VC, _st()), "vit_attn")
    return Case("vit_attn", make, call, ["out"], ["qkv"], ["out"])


# ================================================================================================ letterbox
LB_R = 384


@pytest.fixture(scope="module")
def lb_eng():
    from videollm_online_b200 import tiny_config
    from videollm_online_b200.engine import Engine
    e = Engine(tiny_config(frame_resolution=LB_R), "cuda:0", max_vit_batch=2)
    yield e
    e.close()


def _letterbox_case():
    """one 640 x 480 RGB camera frame on the device.  The canvas is what the previous pass's patchify may still read:
    the kernel must not write it before the wait."""
    W, H = 640, 480

    def make(lib):
        return dict(pixels=torch.randint(0, 256, (H, W, 3), dtype=torch.uint8, device="cuda", generator=_gen(16)),
                    canvas=torch.full((1 + 1, 3, LB_R, LB_R), 0xAB, dtype=torch.uint8, device="cuda"))

    def call(lib, s):
        from videollm_online_b200._lib import VloLetterboxFrame
        eng = s["eng"]
        taps, sw = eng._letterbox_taps(W, H)
        d = (VloLetterboxFrame * 1)()
        d[0].d_pixels, d[0].d_taps, d[0].width, d[0].height = s["pixels"].data_ptr(), taps.data_ptr(), W, H
        d[0].bgr, d[0].x_taps, d[0].y_taps = 0, 0, sw
        _check(eng.lib.vlo_letterbox(eng._h, d, 1, _p(s["canvas"]), _st()), "letterbox")
    return Case("letterbox", make, call, ["canvas"], [Region("pixels", poison=0x5A)], ["canvas"])


# ================================================================================================ the registry
def _cases():
    cs = []
    for shape in DEC_SHAPES:
        for fmt in (FMT_BF16, FMT_F16):
            for mode in (0, 1):
                cs.append(_gemm_ws_case(fmt, mode, shape))
        for fmt in (FMT_E4M3, FMT_E4M3_A8, FMT_I4):
            cs.append(_gemm_ws_q_case(fmt, shape))
        for fmt in (FMT_E4M3, FMT_I4):
            cs.append(_tiles_q_case(fmt, shape))
    for shape in SWIGLU_SHAPES:
        for fmt in (FMT_BF16, FMT_E4M3, FMT_E4M3_A8, FMT_I4):
            cs.append(_swiglu_case(fmt, shape))
    for shape in PREFILL_SHAPES:
        for form in ("bf16", "fp8", "w8a8", "int4"):
            cs.append(_prefill_case(form, shape))
    for shape in VIT_SHAPES:
        cs += [_vit_gemm_case("gemm_vit", shape), _vit_gemm_case("gemm", shape)]
    for shape in ("8b", "tiny"):
        cs += [_resid_case(False, shape), _resid_case(True, shape)]
    cs += [_quant_rows_case(), _qkv_rope_case()]
    cs += [_attn_case("contiguous", 65), _attn_case("contiguous", 13000)]
    for kv in (100, 13020):            # the step's rows share the last block with cached rows
        cs += [_attn_case("paged", kv), _attn_case("segments", kv, [6, 5]), _attn_case("segments", kv, [1, 1, 1, 1])]
    cs += [_decision_case(), _sample_case()]
    cs += [_patchify_case(), _layernorm_case(), _fix_ln_case(), _vit_attn_case(), _letterbox_case()]
    return cs


CASES = _cases()
LATE_IN = [(c, r) for c in CASES for r in c.late_in]
LATE_OUT = [(c, r) for c in CASES for r in c.late_out]
_SERIAL = {}


def _make(case, lib, lb_eng):
    s = case.make(lib)
    if case.name == "letterbox":
        s["eng"] = lb_eng
    torch.cuda.synchronize()
    return s


def _serial(case, lib, lb_eng):
    """the outputs of one plain run on the real operands (no probe armed)"""
    if case.name not in _SERIAL:
        s = _make(case, lib, lb_eng)
        case.call(lib, s)
        torch.cuda.synchronize()
        _SERIAL[case.name] = {n: s[n].clone() for n in case.outs}
    return _SERIAL[case.name]


def _probed(lib, mode, arm, run):
    """arm the probe, run the entry once, and check that exactly this probe ran"""
    n0 = lib.vlo_op_pdl_probe_count()
    _check(lib.vlo_op_pdl_arm(mode, *arm, SPIN_NS), "pdl_arm")
    run()
    n1 = lib.vlo_op_pdl_probe_count()
    assert n0 >= 0 and n1 == n0 + 1, f"the entry did not launch the armed probe ({n0} -> {n1} probes)"


def _plan_check(lib, case):
    """the segmented cases run the plan they are named after"""
    if getattr(case, "segs", None):
        counts = (C.c_int32 * 4)()
        lens = (C.c_int32 * len(case.segs))(*case.segs)
        kv = int(case.name.rsplit("kv", 1)[1])
        _check(lib.vlo_op_attn_plan_counts(len(case.segs), lens, HQ, HK, D, kv, counts), "plan counts")
        assert (counts[1] > 0) if "/cluster/" in case.name else (counts[2] > 0), f"{case.name}: {list(counts)}"


def _diff(case, s, want):
    return [n for n in case.outs if not _same_bits(s[n], want[n])]


# ================================================================================================ controls
CANARY_WORDS = 64 * 256


def _canary(lib, variant, mode):
    """(dst after the run, snapshot or None, old src, real src, old dst)"""
    from videollm_online_b200._lib import PDL_LATE_READ, PDL_LATE_WRITE
    g = _gen(17)
    real = torch.randint(0, 1 << 30, (CANARY_WORDS,), dtype=torch.int32, device="cuda", generator=g)
    old = torch.full_like(real, 0x0BADF00D)
    dst0 = torch.full_like(real, 0x5EED)
    dst = dst0.clone()
    if mode == PDL_LATE_WRITE:
        src, stash = old.clone(), real.clone()
        arm = (_p(src), _p(stash), CANARY_WORDS * 4, 1, 0)
        snap = None
    else:
        src = real.clone()
        snap = dst0.clone()
        arm = (_p(dst), _p(snap), CANARY_WORDS * 4, 1, 0)
    torch.cuda.synchronize()
    _probed(lib, mode, arm, lambda: _check(lib.vlo_op_pdl_canary(variant, _p(src), _p(dst), CANARY_WORDS, _st()),
                                           "canary"))
    return dst, snap, old, real, dst0


def test_canary_that_waits_passes_both_probes(lib):
    from videollm_online_b200._lib import PDL_LATE_READ, PDL_LATE_WRITE
    dst, _, _, real, _ = _canary(lib, 0, PDL_LATE_WRITE)
    assert torch.equal(dst, real), "late write: the canary that waits did not copy the operand's real values"
    dst, snap, _, real, dst0 = _canary(lib, 0, PDL_LATE_READ)
    assert torch.equal(snap, dst0), "late read: the canary that waits wrote before the probe ended"
    assert torch.equal(dst, real)


def test_canary_reading_early_is_caught(lib):
    """the seeded read violation returns the old contents of its input: a kernel reading before its wait cannot pass"""
    from videollm_online_b200._lib import PDL_LATE_WRITE
    dst, _, old, real, _ = _canary(lib, 1, PDL_LATE_WRITE)
    seen = int((dst == old).sum())
    assert seen == CANARY_WORDS, (f"the read-early canary read {CANARY_WORDS - seen} of {CANARY_WORDS} words after the "
                                  f"probe: the probe does not overlap its dependents, so this file could not see a race")


def test_canary_writing_early_is_caught(lib):
    """the seeded write violation shows in the late snapshot of its output"""
    from videollm_online_b200._lib import PDL_LATE_READ
    dst, snap, _, real, dst0 = _canary(lib, 2, PDL_LATE_READ)
    seen = int((snap == real).sum())
    assert seen == CANARY_WORDS, (f"the write-early canary's write of {CANARY_WORDS - seen} of {CANARY_WORDS} words was "
                                  f"missing from the snapshot: the probe does not overlap its dependents")


def test_probe_rejects_bad_arguments(lib):
    from videollm_online_b200._lib import PDL_LATE_WRITE, VloError
    t = torch.zeros(64, dtype=torch.int32, device="cuda")
    for args in [(3, _p(t), _p(t), 256, 1, 0, SPIN_NS), (PDL_LATE_WRITE, _p(t), _p(t), 256, 1, 0, 2_000_001),
                 (PDL_LATE_WRITE, _p(t), _p(t), 256, 1, 0, 0), (PDL_LATE_WRITE, None, _p(t), 256, 1, 0, SPIN_NS),
                 (PDL_LATE_WRITE, _p(t), _p(t), 128, 2, 64, SPIN_NS)]:
        with pytest.raises(VloError):
            _check(lib.vlo_op_pdl_arm(*args), "pdl_arm")


# ================================================================================================ the entries
@pytest.mark.parametrize("case,operand", LATE_IN, ids=[f"{c.name}:{r}" for c, r in LATE_IN])
def test_late_input(lib, lb_eng, case, operand):
    """the operand arrives SPIN_NS after the kernel under test started: the outputs must still be the serial run's"""
    from videollm_online_b200._lib import PDL_LATE_WRITE
    _plan_check(lib, case)
    want = _serial(case, lib, lb_eng)
    s = _make(case, lib, lb_eng)
    reg = case.late_in[operand]
    t = s[reg.name]
    real = t.clone()
    reg.fill(t)
    assert not torch.equal(_bytes(t), _bytes(real)), f"{case.name}: the poison equals the operand"
    torch.cuda.synchronize()
    _probed(lib, PDL_LATE_WRITE, reg.arm_args(t, real), lambda: case.call(lib, s))
    torch.cuda.synchronize()
    if reg.name not in case.outs:       # (an operand the kernel updates in place is compared as an output)
        assert torch.equal(_bytes(t), _bytes(real)), f"{case.name}: the probe did not restore {operand}"
    bad = _diff(case, s, want)
    assert not bad, f"{case.name}: {bad} differ from the serial run when {operand} arrives late: read before the wait"


@pytest.mark.parametrize("case,region", LATE_OUT, ids=[f"{c.name}:{r}" for c, r in LATE_OUT])
def test_late_output(lib, lb_eng, case, region):
    """a snapshot taken SPIN_NS after the kernel under test started must hold what the region held before the launch;
    the outputs are the serial run's"""
    from videollm_online_b200._lib import PDL_LATE_READ
    _plan_check(lib, case)
    want = _serial(case, lib, lb_eng)
    s = _make(case, lib, lb_eng)
    reg = case.late_out[region]
    t = s[reg.name]
    snap = t.clone()                    # the probe's exchange hands the kernel these values
    if reg.marker is not None:
        reg.fill(t, reg.marker)
    before = reg.gather(t).clone()
    torch.cuda.synchronize()
    _probed(lib, PDL_LATE_READ, reg.arm_args(t, snap), lambda: case.call(lib, s))
    torch.cuda.synchronize()
    got = reg.gather(snap)
    changed = int((got != before).sum())
    assert changed == 0, f"{case.name}: {changed} bytes of {region} were written before the wait"
    bad = _diff(case, s, want)
    assert not bad, f"{case.name}: {bad} differ from the serial run"
