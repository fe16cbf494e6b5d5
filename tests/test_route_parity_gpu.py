"""Operator-level parity of the operators whose host code picks a kernel or a launch configuration from the shape: the two bidirectional LSTM
recurrences, the LocalState attention, the fp32 GEMMs and the generic convolution.  Every case calls one C-ABI entry point by name and compares
it with a plain float64 definition written here, at every launch configuration the host can pick and on both sides of every routing threshold.

Which route a GEMM or convolution case took is read from a torch.profiler trace of the call: both sides of a threshold compute the same
numbers, so only the kernel name shows an off-by-one in the dispatch.  The LSTM launch configuration is not visible in a kernel name; a Python
restatement of the host's selection checks that the cases cover every configuration.

Gates (max |got - ref| over the output): tensor-core routes 4e-5 and SIMT GEMM and convolution 1e-5 of max(1, max|ref|, max|pre-activation|),
LocalState 2e-5 of max(1, max|ref|), LSTM 2e-5 absolute (h lies in (-1, 1)).  The GEMM / convolution error follows the size of the sum before the
activation: tanh bounds the output by 1 but not the bf16x3 error of a pre-activation of 5 (2.3e-5, the same in a CPU emulation of the split).
The worst tensor-core case, a K = 64 GEMM, measured 8.2e-6 on an H100; the bf16 hi / lo split emulated on the CPU gives 8.0e-6 for the same
inputs, so that is the scheme's own accuracy and 4e-5 keeps a 4x margin above it.  Outputs are pre-filled with NaN, or with a sentinel where only a
slice is written: every element must come out finite, and every element outside the slice must still hold the sentinel."""
import pytest
import torch
import torch.nn.functional as F
from torch.profiler import ProfilerActivity, profile

pytestmark = pytest.mark.gpu

SENTINEL = 12345.0
ERR_ARG = -1
TC_GATE, SIMT_GATE, LS_GATE, LSTM_GATE = 4e-5, 1e-5, 2e-5, 2e-5

WORST = {}  # family -> largest error seen (scaled as its gate is); printed at the end of the module


@pytest.fixture(scope="module")
def L(lib_built):
    assert torch.cuda.is_available()
    from audio_separator.separator.b200 import _lib

    yield _lib
    print("\nworst error per family: " + ", ".join(f"{k} {v:.2e}" for k, v in sorted(WORST.items())))


def gen(seed):
    return torch.Generator().manual_seed(seed)


def ptr(t, off=0):
    return None if t is None else t.data_ptr() + 4 * off


def stream():
    return torch.cuda.current_stream().cuda_stream


def check_err(got, ref, gate, family, absolute=False, pre=None):
    """max |got - ref| <= gate (absolute) or gate * max(1, max|ref|, max|pre|), pre = the reference before the activation; NaN or inf fails"""
    got = got.detach().cpu().double()
    assert torch.isfinite(got).all(), f"{family}: non-finite output"
    err = (got - ref).abs().max().item()
    scaled = err if absolute else err / max(1.0, ref.abs().max().item(), 0.0 if pre is None else pre.abs().max().item())
    WORST[family] = max(WORST.get(family, 0.0), scaled)
    assert scaled <= gate, f"{family}: error {scaled:.3e} above the gate {gate:.0e}"


def launched_kernels(fn):
    """Run fn under the CUDA profiler; the names of the kernels it launched, without spaces.  The profiler now and then hands back an empty
    trace (2 of several hundred recordings on an H100), so an empty one is recorded again, up to three times; fn writes the same output each time."""
    for _ in range(3):
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            fn()
            torch.cuda.synchronize()
        names = {e.name.replace(" ", "") for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA}
        if names:
            return names
    raise AssertionError("the profiler recorded no CUDA kernel, so the route of this case cannot be checked")


def assert_route(names, want, family):
    """exactly one of the family's kernels ran, and it is `want`"""
    hits = {n for n in names for k in family if k in n}
    assert hits and all(want in n for n in hits), f"expected {want}, the trace has {sorted(hits) or sorted(names)}"


def ACT(y, act):
    return {0: y, 1: F.relu(y), 2: F.gelu(y), 3: F.leaky_relu(y, 0.01), 4: torch.sigmoid(y), 5: torch.tanh(y)}[act]


def strided(buf, shape, strides, off=0):
    return torch.as_strided(buf, shape, strides, off)


def written_mask(n, shape, strides, off=0):
    """boolean mask over a flat buffer of n elements: the elements a strided view covers (asserted not to overlap)"""
    idx = strided(torch.arange(n), shape, strides, off).reshape(-1)
    assert idx.unique().numel() == idx.numel()
    m = torch.zeros(n, dtype=torch.bool)
    m[idx] = True
    return m


# ================================================================================================================ LSTM recurrences
def lstm_ref(xp, whh):
    """xp (2, T, N, 4H) gate pre-activations, whh (2, 4H, H) -> (T, N, 2H) in float64.  Gate order i, f, g, o; direction 1 runs from t = T-1 to 0."""
    xp, whh = xp.double(), whh.double()
    _, T, N, G = xp.shape
    H = G // 4
    out = torch.empty((T, N, 2 * H), dtype=torch.float64)
    for d in range(2):
        h = torch.zeros((N, H), dtype=torch.float64)
        c = torch.zeros((N, H), dtype=torch.float64)
        for s in range(T):
            t = T - 1 - s if d else s
            i, f, g, o = (xp[d, t] + h @ whh[d].t()).split(H, dim=1)
            c = torch.sigmoid(f) * c + torch.sigmoid(i) * torch.tanh(g)
            h = torch.sigmoid(o) * torch.tanh(c)
            out[t, :, d * H : (d + 1) * H] = h
    return out


def lstm_inputs(hid, T, N, seed):
    g = gen(seed)
    xp = torch.randn((2, T, N, 4 * hid), generator=g)  # unit scale: the gates saturate at times
    whh = torch.randn((2, 4 * hid, hid), generator=g) / hid**0.5
    return xp, whh


def wide_lstm_config(hid):
    """The launch selection of b200sep_lstm_bidir_wide_f32 restated (csrc/hdemucs_ops.cu:279-297): cluster size CL, k-split KS, whether
    W_hh^T stays resident in shared memory or is streamed from L2, and the dynamic shared-memory bytes.  None: more than 768 threads per CTA."""
    NS = 8
    CL = next((c for c in (8, 4, 2) if hid % c == 0 and 4 * (hid // c) >= 32), 1)
    UH = hid // CL
    GL = 4 * UH
    if GL > 768:
        return None
    wbytes = hid * GL * 4
    resident = (2 * hid * NS + NS * GL + 2 * NS * UH) * 4 + wbytes <= 200 * 1024
    KS = 1 if resident else next((c for c in (4, 2) if hid % c == 0 and GL * c <= 768), 1)
    smem = (2 * hid * NS + KS * NS * GL + 2 * NS * UH) * 4 + (wbytes if resident else 0)
    return CL, KS, resident, smem


# hid -> (CL, KS, resident): every configuration the host can pick
WIDE_CONFIGS = {7: (1, 1, True), 24: (2, 1, True), 48: (4, 1, True), 64: (8, 1, True), 192: (8, 1, True), 191: (1, 1, False), 384: (8, 4, False),
                512: (8, 2, False), 800: (8, 1, False), 162: (2, 2, False), 198: (2, 1, False), 228: (4, 2, False), 396: (4, 1, False)}
WIDE_CASES = [(hid, 200, 9) for hid in WIDE_CONFIGS] + [(hid, 1, 17) for hid in WIDE_CONFIGS] + [(7, 200, 1), (64, 200, 8), (384, 1, 8), (800, 200, 17)]


def test_lstm_wide_cases_cover_every_configuration():
    for hid, want in WIDE_CONFIGS.items():
        assert wide_lstm_config(hid)[:3] == want, hid
    assert wide_lstm_config(64)[0] * 8 == 64  # UH = 8, the smallest slice
    assert wide_lstm_config(191)[0] == 1 and 4 * 191 == 764
    assert wide_lstm_config(193) is None
    reachable = {c[:3] for c in map(wide_lstm_config, range(1, 4097)) if c}
    assert {wide_lstm_config(h)[:3] for h, _, _ in WIDE_CASES} == reachable and len(reachable) == 12
    for hid in WIDE_CONFIGS:
        assert any(h == hid and N % 8 for h, _, N in WIDE_CASES) and any(h == hid and T == 200 for h, T, _ in WIDE_CASES), hid


@pytest.mark.parametrize("hid,T,N", WIDE_CASES)
def test_lstm_bidir_wide_vs_fp64(L, hid, T, N):
    xp, whh = lstm_inputs(hid, T, N, hid * 1000 + T + N)
    ref = lstm_ref(xp, whh)
    xd, wd = xp.cuda(), whh.transpose(1, 2).contiguous().cuda()  # the kernel takes W_hh^T (2, H, 4H)
    out = torch.full((T, N, 2 * hid), float("nan"), device="cuda")
    L.check(L.lib.b200sep_lstm_bidir_wide_f32(ptr(xd), ptr(wd), ptr(out), T, N, hid, stream()), "lstm_bidir_wide_f32")
    torch.cuda.synchronize()
    check_err(out, ref, LSTM_GATE, "lstm_bidir_wide_f32", absolute=True)


def test_lstm_bidir_wide_rejects_too_many_threads(L):
    x = torch.zeros(2 * 8 * 193, device="cuda")
    w = torch.zeros(2 * 193 * 772, device="cuda")
    out = torch.full((2 * 193,), SENTINEL, device="cuda")
    assert L.lib.b200sep_lstm_bidir_wide_f32(ptr(x), ptr(w), ptr(out), 1, 1, 193, stream()) == ERR_ARG
    torch.cuda.synchronize()
    assert (out.cpu() == SENTINEL).all()


# hid 54 / 55: the shared-memory image (4 H^2 + 5 H floats) on either side of the 48 KB default
VR_LSTM_CASES = [(h, 200, 3) for h in (1, 31, 54, 55, 64, 96)] + [(h, 1, 1) for h in (1, 31, 54, 55, 64, 96)] + [(55, 200, 1), (96, 1, 3)]


@pytest.mark.parametrize("hid,T,N", VR_LSTM_CASES)
def test_lstm_bidir_vs_fp64(L, hid, T, N):
    xp, whh = lstm_inputs(hid, T, N, hid * 1000 + T + N + 7)
    ref = lstm_ref(xp, whh)
    xd, wd = xp.cuda(), whh.cuda()
    out = torch.full((T, N, 2 * hid), float("nan"), device="cuda")
    L.check(L.lib.b200sep_lstm_bidir_f32(ptr(xd), ptr(wd), ptr(out), T, N, hid, stream()), "lstm_bidir_f32")
    torch.cuda.synchronize()
    check_err(out, ref, LSTM_GATE, "lstm_bidir_f32", absolute=True)


def test_lstm_bidir_rejects_hid_97(L):
    x = torch.zeros(2 * 4 * 97, device="cuda")
    w = torch.zeros(2 * 4 * 97 * 97, device="cuda")
    out = torch.full((2 * 97,), SENTINEL, device="cuda")
    assert L.lib.b200sep_lstm_bidir_f32(ptr(x), ptr(w), ptr(out), 1, 1, 97, stream()) == ERR_ARG
    torch.cuda.synchronize()
    assert (out.cpu() == SENTINEL).all()


# ================================================================================================================ LocalState attention
def local_state_ref(q, k, ct, dq, heads, nd):
    """The attention core of LocalState (demucs.py:206-229) in float64: q / k / content (B, C, T), decay logits (B, heads * nd, T)."""
    B, C, T = q.shape
    idx = torch.arange(T, dtype=torch.float64)
    delta = idx[:, None] - idx[None, :]
    qq, kk, cc = (t.double().view(B, heads, -1, T) for t in (q, k, ct))
    dots = torch.einsum("bhct,bhcs->bhts", kk, qq) / kk.shape[2] ** 0.5
    decays = torch.arange(1, nd + 1, dtype=torch.float64)
    dqq = torch.sigmoid(dq.double().view(B, heads, -1, T)) / 2
    dots = dots + torch.einsum("fts,bhfs->bhts", -decays.view(-1, 1, 1) * delta.abs() / nd**0.5, dqq)
    dots.masked_fill_(torch.eye(T, dtype=torch.bool), -100)
    return torch.einsum("bhts,bhct->bhcs", torch.softmax(dots, dim=2), cc).reshape(B, C, T), dots


def run_local_state(L, q, k, ct, dq, heads, nd):
    B, C, T = q.shape
    qd, kd, cd, dd = q.cuda(), k.cuda(), ct.cuda(), dq.cuda()
    out = torch.full((B, C, T), float("nan"), device="cuda")
    L.check(L.lib.b200sep_local_state_attn_f32(ptr(qd), ptr(kd), ptr(cd), ptr(dd), ptr(out), B, C, T, heads, nd, stream()), "local_state_attn_f32")
    torch.cuda.synchronize()
    return out


LS_CH = (1, 2, 3, 4, 6, 8, 12, 16, 24, 32, 48, 64, 96)


def ls_tile(ch):
    return 64 if ch <= 48 else 32  # key positions per tile (R = 2 or 1 per lane)


LS_CASES = []
for _ch in LS_CH:
    _tt = ls_tile(_ch)
    for _T in (1, _tt - 1, _tt, _tt + 1, 2 * _tt + 1):
        _i = len(LS_CASES)
        LS_CASES.append((_ch, _T, (1, 4)[_i % 2], (1, 4)[(_i // 2) % 2], 1 + (_i % 3 == 0)))


@pytest.mark.parametrize("CH,T,heads,nd,B", LS_CASES)
def test_local_state_attn_vs_fp64(L, CH, T, heads, nd, B):
    g = gen(CH * 1000 + T * 10 + heads + nd)
    C = CH * heads
    q, k, ct = (torch.randn((B, C, T), generator=g) for _ in range(3))
    dq = torch.randn((B, heads * nd, T), generator=g) * 2 - 1
    sat = torch.rand(dq.shape, generator=g)
    dq = torch.where(sat < 0.1, torch.full_like(dq, 30.0), torch.where(sat > 0.9, torch.full_like(dq, -30.0), dq))  # sigmoid saturated both ways
    ref, _ = local_state_ref(q, k, ct, dq, heads, nd)
    check_err(run_local_state(L, q, k, ct, dq, heads, nd), ref, LS_GATE, "local_state_attn_f32")


@pytest.mark.parametrize("CH", [16, 64])
def test_local_state_attn_running_max_rescale(L, CH):
    """Scores scaled by 10 with the larger keys in the later tiles and no distance penalty: most rows find their maximum far above everything in
    the first key tile, so the accumulators of the first tile must be rescaled."""
    TT, heads, nd, B = ls_tile(CH), 2, 1, 1
    T, C = 2 * TT + 1, CH * heads
    g = gen(CH + 5)
    q = torch.randn((B, C, T), generator=g) * 10
    k = torch.randn((B, C, T), generator=g)
    k[:, :, TT:] *= 3
    ct = torch.randn((B, C, T), generator=g)
    dq = torch.full((B, heads * nd, T), -30.0)
    ref, dots = local_state_ref(q, k, ct, dq, heads, nd)
    first, later = dots[:, :, :TT].amax(2), dots[:, :, TT:].amax(2)
    assert (later > first + 20).float().mean().item() > 0.75
    check_err(run_local_state(L, q, k, ct, dq, heads, nd), ref, LS_GATE, "local_state_attn_f32")


def test_local_state_attn_rejects_5_channels_per_head(L):
    x = torch.zeros((1, 5, 9), device="cuda")
    d = torch.zeros((1, 1, 9), device="cuda")
    out = torch.full((1, 5, 9), SENTINEL, device="cuda")
    assert L.lib.b200sep_local_state_attn_f32(ptr(x), ptr(x), ptr(x), ptr(d), ptr(out), 1, 5, 9, 1, 1, stream()) == ERR_ARG
    torch.cuda.synchronize()
    assert (out.cpu() == SENTINEL).all()


# ================================================================================================================ GEMM
GEMM_KERNELS = ("tc_f32_kernel", "gemm_small_n_kernel", "gemm_f32_kernel")
TC, SN8, SN16, SIMT = "tc_f32_kernel", "gemm_small_n_kernel<8>", "gemm_small_n_kernel<16>", "gemm_f32_kernel"


def c4(n):
    return -(-n // 4) * 4


def gemm_check(L, route, M, N, K, batch=1, lda=None, ldb=None, ldc=None, a_off=0, sA=None, sB=None, sC=None, alpha=1.0, bias_n=False, bias_m=False, act=0,
               res=False, rs=False, packed=False, kn=False):
    """C[z] = act(alpha * A[z] B[z]^T + bias_n + bias_m), then res + res_scale * C.  B is (N, K) rows of ldb, or (K, N) rows of ldb with kn
    (b200sep_gemm_kn_f32).  C and res share ldc / sC; everything C's view does not cover must keep the sentinel."""
    g = gen(M * 7 + N * 3 + K + batch + act + 100 * a_off + 1000 * kn)
    lda = lda or K
    ldb = ldb or (N if kn else K)
    ldc = ldc or N
    sA = M * lda + 4 if sA is None else sA
    b_rows, b_cols = (K, N) if kn else (N, K)
    sB = b_rows * ldb + 8 if sB is None else sB
    sC = M * ldc + 4 if sC is None else sC
    nA, nB, nC = a_off + (batch - 1) * sA + (M - 1) * lda + K, (batch - 1) * sB + (b_rows - 1) * ldb + b_cols, (batch - 1) * sC + (M - 1) * ldc + N
    Ab, Bb = torch.randn(nA, generator=g), torch.randn(nB, generator=g) / K**0.5
    A = strided(Ab, (batch, M, K), (sA, lda, 1), a_off).double()
    Bm = strided(Bb, (batch, b_rows, b_cols), (sB, ldb, 1)).double()
    y = alpha * (A @ Bm if kn else A @ Bm.transpose(1, 2))
    bn = torch.randn(N, generator=g) if bias_n else None
    bm = torch.randn(M, generator=g) if bias_m else None
    if bn is not None:
        y = y + bn.double()
    if bm is not None:
        y = y + bm.double()[:, None]
    pre = y
    y = ACT(y, act)
    Rb = torch.randn(nC, generator=g) if res else None
    scale = torch.rand(N, generator=g) + 0.5 if rs else None
    if res:
        y = strided(Rb, (batch, M, N), (sC, ldc, 1)).double() + (scale.double() if rs else 1.0) * y
    Ad, Bd, Cd = Ab.cuda(), Bb.cuda(), torch.full((nC,), SENTINEL, device="cuda")
    bnd, bmd, Rd, sd = (None if t is None else t.cuda() for t in (bn, bm, Rb, scale))
    pk = None
    if packed:
        pk = torch.empty(L.lib.b200sep_tc_packed_floats(N, K), device="cuda")
        L.check(L.lib.b200sep_tc_pack_linear_weights(ptr(Bd), N, K, ldb, ptr(pk), stream()), "tc_pack_linear_weights")
    if kn:
        call = lambda: L.check(L.lib.b200sep_gemm_kn_f32(ptr(Ad, a_off), ptr(Bd), ptr(Cd), M, N, K, lda, ldb, ldc, batch, sA, sB, sC, alpha, stream()), "gemm_kn_f32")
    else:
        call = lambda: L.check(L.lib.b200sep_gemm_f32(ptr(Ad, a_off), ptr(Bd), ptr(Cd), M, N, K, lda, ldb, ldc, batch, sA, sB, sC, alpha, ptr(bnd), ptr(bmd), act,
                                                     ptr(Rd), ptr(sd), ptr(pk), stream()), "gemm_f32")
    assert_route(launched_kernels(call), route, GEMM_KERNELS)
    got = Cd.cpu()
    m = written_mask(nC, (batch, M, N), (sC, ldc, 1))
    assert (got[~m] == SENTINEL).all(), "an element outside C's view was written"
    check_err(strided(got, (batch, M, N), (sC, ldc, 1)), y, TC_GATE if route == TC else SIMT_GATE, ("gemm_kn_f32 " if kn else "gemm_f32 ") + ("tc" if route == TC else "simt"), pre=pre)


# (M, N, K, batch) -> route, both sides of every threshold of tc_gemm_usable (K >= 32, N >= 32, M N batch >= 16384) and of the small-N kernel
# (N <= 16, M >= 1024)
GEMM_THRESHOLDS = [
    ((128, 128, 31, 1), SIMT), ((128, 128, 32, 1), TC),
    ((600, 31, 64, 1), SIMT), ((600, 32, 64, 1), TC),
    ((127, 129, 64, 1), SIMT), ((128, 128, 64, 1), TC),
    ((64, 64, 64, 3), SIMT), ((64, 64, 64, 4), TC),
] + [((M, N, 67, 1), (SN8 if N <= 8 else SN16) if (M >= 1024 and N <= 16) else SIMT) for N in (1, 8, 9, 16, 17) for M in (1023, 1024)]


@pytest.mark.parametrize("shape,route", GEMM_THRESHOLDS)
def test_gemm_route_thresholds(L, shape, route):
    M, N, K, batch = shape
    gemm_check(L, route, M, N, K, batch=batch, bias_n=True, act=2)


# every route: float4 and scalar loads (K % 4 tails with a float4-aligned lda, lda % 4 != 0, A one float off alignment), every epilogue, batches
ROUTE_SHAPES = {TC: (200, 96, 64), SN8: (1100, 5, 64), SN16: (1030, 13, 64), SIMT: (150, 40, 20)}
GEMM_VARIANTS = {
    "float4": dict(act=0),
    "k%4=1": dict(dk=1, act=5, bias_n=True),
    "k%4=2": dict(dk=2, act=4, bias_m=True),
    "k%4=3": dict(dk=3, act=3, bias_n=True, bias_m=True, alpha=0.5),
    "lda%4=3": dict(lda_pad=3, act=1, res=True),
    "a+1": dict(a_off=1, act=2, res=True, rs=True, ldc_pad=3),
    "batch3": dict(batch=3, act=5, res=True, rs=True, bias_n=True, bias_m=True, alpha=-1.25, ldc_pad=2),
    "packed_sB0": dict(batch=2, sB=0, packed=True, act=0, bias_n=True),
}


@pytest.mark.parametrize("variant", list(GEMM_VARIANTS))
@pytest.mark.parametrize("route", [TC, SN8, SN16, SIMT])
def test_gemm_loads_and_epilogues(L, route, variant):
    M, N, K = ROUTE_SHAPES[route]
    v = dict(GEMM_VARIANTS[variant])
    K += v.pop("dk", 0)
    lda = c4(K) + v.pop("lda_pad", 0)  # a multiple of 4 keeps the float4 path unless lda_pad / a_off break it
    ldc = N + v.pop("ldc_pad", 0)
    gemm_check(L, route, M, N, K, lda=lda, ldb=c4(K), ldc=ldc, **v)


# (M, N, K, ldb, ldc, route): B given as (K, N) rows; batch strides, ldb > N, ldc > N
GEMM_KN_CASES = [(100, 20, 30, 25, 23, SIMT), (150, 40, 20, 44, 41, SIMT), (200, 80, 72, 84, 83, TC), (300, 96, 45, 99, 97, TC)]


@pytest.mark.parametrize("M,N,K,ldb,ldc,route", GEMM_KN_CASES)
def test_gemm_kn_routes(L, M, N, K, ldb, ldc, route):
    gemm_check(L, route, M, N, K, batch=2, lda=K + 1, ldb=ldb, ldc=ldc, alpha=0.75, kn=True)


# ================================================================================================================ convolution
CONV_KERNELS = ("tc_f32_kernel", "conv_gen_kernel", "conv_direct_kernel")


def ceil48(n):
    return -(-n // 48) * 48


def block_weight(w):
    """(Cout, Cin, KH, KW) -> [Cin][KH * KW][ceil48(Cout)]"""
    co, ci, kh, kw = w.shape
    out = torch.zeros((ci, kh * kw, ceil48(co)))
    out[:, :, :co] = w.permute(1, 2, 3, 0).reshape(ci, kh * kw, co)
    return out


def gen_route(k, s, dw):
    return "conv_gen_kernel<%d,%d,%d,%d,%d>" % (k[0], k[1], s[0], s[1], dw)


def conv_call(L, x, wb, bias, add, y, B, Cin, H, W, Cout, Ho, Wo, k, s, p, d, act, before, up_axis=0, up=1, trim=0, out_len=0, oct_=0, ooff=0, pk=None):
    return L.lib.b200sep_conv2d_f32(ptr(x), ptr(wb), ptr(bias), ptr(add), ptr(y), B, Cin, H, W, Cout, Ho, Wo, k[0], k[1], s[0], s[1], p[0], p[1], d[0], d[1], act,
                                    int(before), up_axis, up, trim, out_len, oct_, ooff, ptr(pk), stream())


def conv_check(L, route, B, Cin, Cout, hw, k, s=(1, 1), p=(0, 0), d=(1, 1), act=0, add=None, out_c=None, packed=False):
    """y = act(conv2d(x) + bias (+ add before the activation)) (+ add after it), written into channels [off, off + Cout) of an (B, total, Ho, Wo)
    output when out_c = (total, off)."""
    H, W = hw
    g = gen(B * 131 + Cin * 17 + Cout * 5 + H + W + k[0] * 3 + k[1] + act)
    x = torch.randn((B, Cin, H, W), generator=g)
    w = torch.randn((Cout, Cin) + tuple(k), generator=g) / (Cin * k[0] * k[1]) ** 0.5
    b = torch.randn(Cout, generator=g)
    y = F.conv2d(x.double(), w.double(), b.double(), stride=s, padding=p, dilation=d)
    Ho, Wo = y.shape[2:]
    a = torch.randn(y.shape, generator=g) if add else None
    if add == "before":
        y = y + a.double()
    pre = y
    y = ACT(y, act)
    if add == "after":
        y = y + a.double()
    total, off = out_c or (Cout, 0)
    xd, wd, bd, ad = x.cuda(), block_weight(w).cuda(), b.cuda(), (a.cuda() if add else None)
    out = torch.full((B, total, Ho, Wo), SENTINEL if out_c else float("nan"), device="cuda")
    pk = None
    if packed:
        cin8 = -(-Cin // 8) * 8
        pk = torch.empty(L.lib.b200sep_tc_packed_floats(Cout, cin8 * k[0] * k[1]), device="cuda")
        L.check(L.lib.b200sep_tc_pack_conv_weights(ptr(wd), Cin, k[0] * k[1], Cout, ptr(pk), stream()), "tc_pack_conv_weights")
    call = lambda: L.check(conv_call(L, xd, wd, bd, ad, out, B, Cin, H, W, Cout, Ho, Wo, k, s, p, d, act, add == "before", oct_=total if out_c else 0, ooff=off, pk=pk),
                           "conv2d_f32")
    assert_route(launched_kernels(call), route, CONV_KERNELS)
    got = out.cpu()
    if out_c:
        assert (got[:, :off] == SENTINEL).all() and (got[:, off + Cout :] == SENTINEL).all(), "a channel outside the slice was written"
    check_err(got[:, off : off + Cout], y, TC_GATE if route == TC else SIMT_GATE, "conv2d_f32 " + ("tc" if route == TC else "simt"), pre=pre)


# the nine conv_gen tiles and the direct kernel: Cout 50 (two 48-channel tiles), Wo 130 (two 128-wide tiles), 11 input channels (a ragged 8-channel
# chunk), B Ho Wo = 390 < 512 keeps them off the tensor cores
SIMT_CONV_CASES = [
    dict(k=(1, 1), s=(1, 1), p=(0, 0), hw=(3, 130), act=0),
    dict(k=(3, 3), s=(1, 1), p=(1, 1), hw=(3, 130), act=1, add="before"),
    dict(k=(3, 3), s=(2, 2), p=(1, 1), hw=(6, 259), act=2, add="after"),
    dict(k=(1, 3), s=(1, 1), p=(0, 1), hw=(3, 130), act=3, out_c=(61, 7)),
    dict(k=(1, 3), s=(1, 1), p=(0, 2), d=(1, 2), hw=(3, 130), act=4),
    dict(k=(8, 1), s=(4, 1), p=(2, 0), hw=(13, 130), act=5),
    dict(k=(1, 8), s=(1, 4), p=(0, 2), hw=(3, 520), act=5, add="before"),
    dict(k=(2, 1), s=(1, 1), p=(1, 0), hw=(2, 130), act=2, add="after"),
    dict(k=(1, 2), s=(1, 1), p=(0, 1), hw=(3, 129), act=1),
    dict(k=(3, 5), s=(1, 2), p=(2, 2), d=(2, 1), hw=(3, 259), act=5, add="after"),
]


def _simt_conv_id(c):
    return "x".join(map(str, c["k"])) + "s" + "x".join(map(str, c["s"])) + "d" + "x".join(map(str, c.get("d", (1, 1))))


@pytest.mark.parametrize("case", SIMT_CONV_CASES, ids=_simt_conv_id)
def test_conv2d_simt_geometries(L, case):
    c = dict(case)
    route = "conv_direct_kernel" if c.get("d", (1, 1))[0] != 1 else gen_route(c["k"], c["s"], c.get("d", (1, 1))[1])
    conv_check(L, route, 1, 11, 50, **c)


# tc_conv_usable: Cin KH KW >= 32, Cout >= 16, B Ho Wo >= 512 -- exactly on each edge, one below each, and the tensor-core epilogues
TC_CONV_CASES = [
    (dict(B=1, Cin=32, Cout=16, hw=(8, 64), k=(1, 1), act=5), TC),
    (dict(B=1, Cin=31, Cout=16, hw=(8, 64), k=(1, 1), act=5), gen_route((1, 1), (1, 1), 1)),
    (dict(B=1, Cin=32, Cout=15, hw=(8, 64), k=(1, 1), act=5), gen_route((1, 1), (1, 1), 1)),
    (dict(B=1, Cin=32, Cout=16, hw=(7, 73), k=(1, 1), act=5), gen_route((1, 1), (1, 1), 1)),
    (dict(B=2, Cin=32, Cout=16, hw=(4, 64), k=(1, 1), act=1), TC),
    (dict(B=1, Cin=4, Cout=20, hw=(8, 260), k=(1, 8), s=(1, 4), p=(0, 2), act=2), TC),
    (dict(B=1, Cin=3, Cout=20, hw=(8, 260), k=(1, 8), s=(1, 4), p=(0, 2), act=2), gen_route((1, 8), (1, 4), 1)),
    (dict(B=2, Cin=20, Cout=40, hw=(20, 70), k=(3, 3), p=(1, 1), act=5, add="before", packed=True), TC),
    (dict(B=2, Cin=20, Cout=40, hw=(20, 70), k=(3, 3), p=(1, 1), act=2, add="after"), TC),
    (dict(B=1, Cin=48, Cout=33, hw=(30, 50), k=(1, 1), act=1, out_c=(50, 10), packed=True), TC),
]


@pytest.mark.parametrize("case,route", TC_CONV_CASES)
def test_conv2d_tensor_core_edges(L, case, route):
    conv_check(L, route, **case)


def convtr_check(L, route, B, Cin, cout, hw, axis, up, trim, out_len, act, packed=False):
    """nn.ConvTranspose with kernel 2 * up and stride up along axis (1 = H, 2 = W), cropped to [trim, trim + out_len), as the 2-tap convolution
    over the coarse index whose GEMM column r * cout + c produces output sample q * up + r."""
    H, W = hw
    g = gen(B * 7 + Cin + cout + H + W + axis + up)
    x = torch.randn((B, Cin, H, W), generator=g)
    w = torch.randn((Cin, cout, 2 * up), generator=g) / Cin**0.5
    b = torch.randn(cout, generator=g)
    if axis == 1:
        y = F.conv_transpose2d(x.double(), w.double()[:, :, :, None], b.double(), stride=(up, 1))[:, :, trim : trim + out_len]
        k, p, Ho, Wo = (2, 1), (1, 0), H + 1, W
    else:
        y = F.conv_transpose2d(x.double(), w.double()[:, :, None, :], b.double(), stride=(1, up))[:, :, :, trim : trim + out_len]
        k, p, Ho, Wo = (1, 2), (0, 1), H, W + 1
    assert y.shape[axis + 1] == out_len
    pre = y
    y = ACT(y, act)
    wb = torch.zeros((Cin, 2, ceil48(up * cout)))
    for r in range(up):
        wb[:, 0, r * cout : (r + 1) * cout] = w[:, :, r + up]
        wb[:, 1, r * cout : (r + 1) * cout] = w[:, :, r]
    xd, wd, bd = x.cuda(), wb.cuda(), b.cuda()
    out = torch.full(tuple(y.shape), float("nan"), device="cuda")
    pk = None
    if packed:
        pk = torch.empty(L.lib.b200sep_tc_packed_floats(up * cout, -(-Cin // 8) * 8 * 2), device="cuda")
        L.check(L.lib.b200sep_tc_pack_conv_weights(ptr(wd), Cin, 2, up * cout, ptr(pk), stream()), "tc_pack_conv_weights")
    call = lambda: L.check(conv_call(L, xd, wd, bd, None, out, B, Cin, H, W, up * cout, Ho, Wo, k, (1, 1), p, (1, 1), act, False, axis, up, trim, out_len, pk=pk),
                           "conv2d_f32 (transposed)")
    assert_route(launched_kernels(call), route, CONV_KERNELS)
    check_err(out, y, TC_GATE if route == TC else SIMT_GATE, "conv2d_f32 " + ("tc" if route == TC else "simt"), pre=pre)


# (B, Cin, cout, (H, W), axis, up, trim, out_len, act, route): odd out_len, non-zero trim; cout % 16 != 0 keeps the SIMT tiles
CONVTR_CASES = [
    (2, 12, 10, (40, 20), 1, 4, 2, 157, 2, gen_route((2, 1), (1, 1), 1)),
    (2, 12, 10, (3, 150), 2, 4, 2, 597, 5, gen_route((1, 2), (1, 1), 1)),
    (1, 24, 16, (30, 20), 1, 4, 2, 121, 5, TC),
    (1, 24, 16, (4, 150), 2, 4, 3, 599, 2, TC),
]


@pytest.mark.parametrize("B,Cin,cout,hw,axis,up,trim,out_len,act,route", CONVTR_CASES)
def test_conv2d_transposed_routes(L, B, Cin, cout, hw, axis, up, trim, out_len, act, route):
    convtr_check(L, route, B, Cin, cout, hw, axis, up, trim, out_len, act, packed=route == TC)


# ================================================================================================================ a second device in one process
def _device_calls(L):
    """One call per launch site that raises a kernel's dynamic shared-memory limit, on the current device; the outputs, on the host."""
    import mdx_oracle as O
    from audio_separator.separator.b200 import engine, mdx_weights

    outs = {}

    def dev(t):
        return t.contiguous().cuda()

    def done(name, rc, y):
        L.check(rc, name)
        torch.cuda.synchronize()
        outs[name] = y.cpu()

    g = gen(1)
    xp, whh = lstm_inputs(384, 5, 3, 1)
    xd, wd = dev(xp), dev(whh.transpose(1, 2))
    y = torch.empty((5, 3, 768), device="cuda")
    done("lstm_bidir_wide_f32", L.lib.b200sep_lstm_bidir_wide_f32(ptr(xd), ptr(wd), ptr(y), 5, 3, 384, stream()), y)
    xp, whh = lstm_inputs(64, 5, 2, 2)
    xd, wd = dev(xp), dev(whh)
    y = torch.empty((5, 2, 128), device="cuda")
    done("lstm_bidir_f32", L.lib.b200sep_lstm_bidir_f32(ptr(xd), ptr(wd), ptr(y), 5, 2, 64, stream()), y)
    a, b = dev(torch.randn((128, 128), generator=g)), dev(torch.randn((128, 128), generator=g))
    y = torch.empty((128, 128), device="cuda")
    done("gemm_f32", L.lib.b200sep_gemm_f32(ptr(a), ptr(b), ptr(y), 128, 128, 128, 128, 128, 128, 1, 0, 0, 0, 1.0, None, None, 0, None, None, None, stream()), y)
    x = dev(torch.randn((1, 5, 13, 130), generator=g))  # conv_gen_kernel<8, 1, 4, 1, 1>: 64.5 KB of shared memory
    wb = dev(block_weight(torch.randn((20, 5, 8, 1), generator=g)))
    y = torch.empty((1, 20, 3, 130), device="cuda")
    done("conv2d_f32", conv_call(L, x, wb, None, None, y, 1, 5, 13, 130, 20, 3, 130, (8, 1), (4, 1), (2, 0), (1, 1), 0, False), y)
    for name, (B, C, Fr, Lx, hid) in {"dconv_f32 row": (1, 48, 3, 700, 6), "dconv_f32": (1, 192, 1, 300, 24)}.items():
        d = [dev(t) for t in (torch.randn((B, C, Fr, Lx), generator=g), torch.randn((hid, C, 3), generator=g) / (3 * C) ** 0.5, torch.randn(hid, generator=g),
                              torch.rand(hid, generator=g) + 0.5, torch.randn(hid, generator=g), torch.randn((2 * C, hid), generator=g) / hid**0.5,
                              torch.randn(2 * C, generator=g), torch.rand(2 * C, generator=g) + 0.5, torch.randn(2 * C, generator=g), torch.rand(C, generator=g))]
        y = torch.empty_like(d[0])
        work = torch.empty(L.lib.b200sep_dconv_work_floats(B, C, Fr, Lx, hid), device="cuda")
        done(name, L.lib.b200sep_dconv_f32(ptr(d[0]), ptr(y), *[ptr(t) for t in d[1:]], B, C, Fr, Lx, hid, 1, None, ptr(work), stream()), y)
    Lq, Hh = 200, 2
    q, k, v = (dev(torch.randn((1, Lq, Hh * 64), generator=g)) for _ in range(3))
    y = torch.empty((1, Lq, Hh * 64), device="cuda")
    work = torch.empty(L.lib.b200sep_attention_work_floats(1, Hh, Lq, Lq), device="cuda")
    D = Hh * 64
    done("attention_f32", L.lib.b200sep_attention_f32(ptr(q), ptr(k), ptr(v), ptr(y), 1, Hh, Lq, Lq, 64, Lq * D, D, Lq * D, D, Lq * D, D, Lq * D, D, 0.125, 1, ptr(work),
                                                      stream()), y)
    scale, shift = dev(torch.rand(16, generator=g) + 0.5), dev(torch.randn(16, generator=g) * 0.1)
    a, w = dev(torch.randn((256, 64), generator=g)), dev(torch.randn((128, 64), generator=g) / 8)
    y = torch.empty((256, 128), device="cuda")
    done("selftest_umma_gemm", L.lib.b200sep_selftest_umma_gemm(ptr(a), ptr(w), None, ptr(y), 256, 128, 64, 32, 8, ptr(scale), ptr(shift), 1, stream()), y)
    x = dev(torch.randn((1, 16, 4, 128), generator=g))
    wh = (torch.randn((16, 16, 3, 3), generator=g) / 12).contiguous()  # host weights
    y = torch.empty((1, 16, 4, 128), device="cuda")
    done("selftest_umma_conv3x3", L.lib.b200sep_selftest_umma_conv3x3(ptr(x), wh.data_ptr(), ptr(y), 1, 16, 16, 4, 128, ptr(scale), ptr(shift), 1, stream()), y)
    x = dev(torch.randn((1, 32, 4, 128), generator=g))
    wh = (torch.randn((32, 16, 2, 2), generator=g) / 11).contiguous()
    y = torch.empty((1, 16, 8, 256), device="cuda")
    done("selftest_umma_updown", L.lib.b200sep_selftest_umma_updown(ptr(x), wh.data_ptr(), None, ptr(y), 1, 32, 16, 4, 128, ptr(scale), ptr(shift), 1, 1, stream()), y)
    cfg = O.MDXConfig(n_fft=1536, hop_length=256, dim_f=768, dim_t=32, segment_size=32, g=8)
    w = O.make_convtdfnet_weights(cfg, seed=7, out_gain=0.05)
    hp = mdx_weights.infer_hparams_from_state(w)
    net = engine.MdxNet(mdx_weights.flatten_state(w, **hp), dim_t=cfg.dim_t, max_batch=1, precision=0, **hp)  # the fp32 SIMT convolutions
    outs["mdxnet precision 0"] = net.forward(dev(torch.randn((1, 4, cfg.dim_f, cfg.dim_t), generator=g))).cpu()
    del net
    return outs


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two CUDA devices")
def test_kernels_on_a_second_device_in_one_process(L):
    """A kernel attribute (the dynamic shared-memory limit) belongs to the function in one device's context: after a call on cuda:0, the first
    call on cuda:1 must still set it there.  Every result on cuda:1 must equal the cuda:0 result bit for bit."""
    torch.cuda.set_device(0)
    first = _device_calls(L)
    try:
        torch.cuda.set_device(1)
        second = _device_calls(L)
    finally:
        torch.cuda.set_device(0)
    assert first.keys() == second.keys()
    for name in first:
        assert torch.equal(first[name], second[name]), name
