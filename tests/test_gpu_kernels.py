"""GPU parity of the libdmlb kernels against the oracle (oracle/*) — called through the C ABI.

Bit-exact where the arithmetic is integer / byte / order-defined (casts, scales, min/max, counters, gathers, the
rank-ordered sums); toleranced (stated per test) where the summation order differs from the reference's.
"""
import ctypes

import numpy as np
import pytest
import torch

from conftest import load_json, load_npz
from oracle import grad_oracle

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module')
def lib():
    from dmlcloud_b200 import _native as N

    return N.cuda_lib(0)


def N_():
    from dmlcloud_b200 import _native as N

    return N


def sptr():
    return N_().stream_ptr()


def rand_grads(n, seed):
    rng = np.random.RandomState(seed)
    g = rng.randn(n).astype(np.float32) * (10.0 ** rng.randint(-6, 3, n)).astype(np.float32)
    if n:
        g[rng.randint(0, n, max(1, n // 50))] = 0.0
    return g


SIZES = [0, 1, 3, 4, 5, 7, 8, 31, 1023, 1024, 1025, 4160, 10330, 513000, (1 << 20) + 3]


class TestBucketKernels:
    @pytest.mark.parametrize('n', SIZES)
    @pytest.mark.parametrize('world', [1, 3, 8])
    def test_scale_inplace_bit_exact(self, lib, n, world):
        g = rand_grads(n, n + world)
        t = torch.from_numpy(g.copy()).cuda()
        N_().check(lib.dmlb_bucket_scale_f32(t.data_ptr(), n, 1.0 / world, sptr()))
        assert (t.cpu().numpy() == grad_oracle.scale_f32(g, world)).all()

    @pytest.mark.parametrize('n', SIZES)
    def test_pack_unpack_bf16_bit_exact(self, lib, n):
        g = rand_grads(n, n)
        src = torch.from_numpy(g).cuda()
        wire = torch.zeros(n + 8, dtype=torch.bfloat16, device='cuda')
        N_().check(lib.dmlb_bucket_pack_f32_bf16(src.data_ptr(), wire.data_ptr(), n, 0.125, sptr()))
        want_bits = grad_oracle.f32_to_bf16_bits(grad_oracle.scale_f32(g, 8))
        got_bits = wire[:n].view(torch.int16).cpu().numpy().view(np.uint16)
        assert (got_bits == want_bits).all()
        assert (wire[n:].float().cpu().numpy() == 0).all()  # nothing written past n
        out = torch.full((n + 4,), -7.0, device='cuda')
        sumsq = torch.zeros(1, dtype=torch.float64, device='cuda')
        N_().check(lib.dmlb_bucket_unpack_bf16_f32(wire.data_ptr(), out.data_ptr(), n, 1.0, sumsq.data_ptr(), sptr()))
        want = grad_oracle.bf16_bits_to_f32(want_bits)
        assert (out[:n].cpu().numpy() == want).all() and (out[n:].cpu().numpy() == -7.0).all()
        np.testing.assert_allclose(sumsq.item(), np.sum(want.astype(np.float64) ** 2), rtol=1e-12)

    @pytest.mark.parametrize('n', SIZES)
    def test_round_bf16_inplace_equals_pack_then_unpack(self, lib, n):
        g = rand_grads(n, 77 + n)
        t = torch.from_numpy(g.copy()).cuda()
        sumsq = torch.zeros(1, dtype=torch.float64, device='cuda')
        N_().check(lib.dmlb_bucket_round_bf16_f32(t.data_ptr(), n, 0.25, sumsq.data_ptr(), sptr()))
        want = grad_oracle.round_bf16(grad_oracle.scale_f32(g, 4))
        assert (t.cpu().numpy() == want).all()
        np.testing.assert_allclose(sumsq.item(), np.sum(want.astype(np.float64) ** 2), rtol=1e-12)

    @pytest.mark.parametrize('n', [0, 5, 4095, 4096, 4097, 3 * 4096, 600 * 4096 + 17, 11_689_512])
    def test_tma_pack_variant_is_bit_identical(self, lib, n):
        g = rand_grads(n, 5 + n)
        src = torch.from_numpy(g).cuda()
        a = torch.zeros(n + 8, dtype=torch.bfloat16, device='cuda')
        b = torch.zeros(n + 8, dtype=torch.bfloat16, device='cuda')
        N_().check(lib.dmlb_bucket_pack_f32_bf16_regs(src.data_ptr(), a.data_ptr(), n, 0.125, sptr()))
        N_().check(lib.dmlb_bucket_pack_f32_bf16_tma(src.data_ptr(), b.data_ptr(), n, 0.125, sptr()))
        assert torch.equal(a.view(torch.int16), b.view(torch.int16))
        want = grad_oracle.f32_to_bf16_bits(grad_oracle.scale_f32(g, 8))
        assert (b[:n].view(torch.int16).cpu().numpy().view(np.uint16) == want).all()
        # K2: TMA bulk load + bulk store vs the register path vs the oracle
        x = torch.full((n + 4,), -3.0, device='cuda')
        y = torch.full((n + 4,), -3.0, device='cuda')
        N_().check(lib.dmlb_bucket_unpack_bf16_f32_regs(b.data_ptr(), x.data_ptr(), n, 2.0, None, sptr()))
        N_().check(lib.dmlb_bucket_unpack_bf16_f32_tma(b.data_ptr(), y.data_ptr(), n, 2.0, sptr()))
        assert torch.equal(x, y)
        assert (y[:n].cpu().numpy() == grad_oracle.bf16_bits_to_f32(want) * np.float32(2.0)).all()
        assert (y[n:].cpu().numpy() == -3.0).all()

    @pytest.mark.parametrize('offset', [1, 2, 3])
    def test_misaligned_pointers_take_the_safe_path(self, lib, offset):
        n = 5000
        g = rand_grads(n + 8, 3)
        base = torch.from_numpy(g).cuda()
        src = base[offset:offset + n]  # 4-byte aligned only
        dst = torch.zeros(n + 8, device='cuda')[offset:offset + n]
        N_().check(lib.dmlb_bucket_pack_f32_f32(src.data_ptr(), dst.data_ptr(), n, 0.5, sptr()))
        assert (dst.cpu().numpy() == g[offset:offset + n] * np.float32(0.5)).all()
        wire = torch.zeros(n + 8, dtype=torch.bfloat16, device='cuda')[1:1 + n]  # 2-byte aligned: scalar fallback
        N_().check(lib.dmlb_bucket_pack_f32_bf16(src.data_ptr(), wire.data_ptr(), n, 1.0, sptr()))
        got = wire.view(torch.int16).cpu().numpy().view(np.uint16)
        assert (got == grad_oracle.f32_to_bf16_bits(g[offset:offset + n])).all()

    def test_special_values(self, lib):
        g = np.array([0.0, -0.0, np.inf, -np.inf, np.nan, 1e-45, -1e-45, 3.3895314e38, 1.0, 1.0039062, 1.0117188, 7],
                     dtype=np.float32)
        src = torch.from_numpy(g).cuda()
        wire = torch.zeros(len(g), dtype=torch.bfloat16, device='cuda')
        N_().check(lib.dmlb_bucket_pack_f32_bf16(src.data_ptr(), wire.data_ptr(), len(g), 1.0, sptr()))
        want = src.to(torch.bfloat16)  # torch's RNE cast is the reference's cast (default_hooks.py:57)
        assert (wire.view(torch.int16) == want.view(torch.int16)).all()

    @pytest.mark.parametrize('n', [1, 5, 10330, 700001])
    def test_sumsq_and_clip(self, lib, n):
        g = (np.random.RandomState(n).randn(n) * 3).astype(np.float32)
        t = torch.from_numpy(g.copy()).cuda()
        sumsq = torch.zeros(1, dtype=torch.float64, device='cuda')
        N_().check(lib.dmlb_bucket_sumsq_f32(t.data_ptr(), n, sumsq.data_ptr(), sptr()))
        coef, total = grad_oracle.clip_coef(g, 1.5)
        np.testing.assert_allclose(np.sqrt(sumsq.item()), total, rtol=1e-12)
        N_().check(lib.dmlb_bucket_clip_f32(t.data_ptr(), n, sumsq.data_ptr(), 1.5, sptr()))
        want = g * np.float32(min(1.0, np.float32(1.5) / (np.float32(total) + np.float32(1e-6))))
        np.testing.assert_allclose(t.cpu().numpy(), want, rtol=3e-7, atol=0)  # one fp32 ulp on the coefficient

    def test_clip_matches_torch_clip_grad_norm(self, lib):
        from dmlcloud_b200.gradsync import clip_grad_norm_

        torch.manual_seed(0)
        ps = [torch.nn.Parameter(torch.randn(s, device='cuda')) for s in ((7, 5), (129,), (1,), (64, 64))]
        ref = [torch.nn.Parameter(p.detach().clone()) for p in ps]
        for p, r in zip(ps, ref):
            p.grad = torch.randn_like(p) * 4
            r.grad = p.grad.clone()
        norm = clip_grad_norm_(ps, 0.75)
        ref_norm = torch.nn.utils.clip_grad_norm_(ref, 0.75)
        torch.testing.assert_close(norm, ref_norm, rtol=1e-6, atol=0)
        for p, r in zip(ps, ref):
            torch.testing.assert_close(p.grad, r.grad, rtol=1e-6, atol=1e-9)

    def test_multi_tensor_pack_unpack(self, lib):
        N = N_()
        shapes = [(16, 1, 3, 3), (16,), (16, 16, 3, 3), (16,), (10, 784), (10,), (3,), (1,)]  # MNIST CNN + odd tails
        rng = np.random.RandomState(0)
        grads = [torch.from_numpy(rng.randn(*s).astype(np.float32)).cuda() for s in shapes]
        total = sum(g.numel() for g in grads)
        segs = (N.Seg * len(grads))()
        off = 0
        for i, g in enumerate(grads):
            segs[i] = N.Seg(g.data_ptr(), off, g.numel())
            off += g.numel()
        dsegs = torch.frombuffer(bytearray(bytes(segs)), dtype=torch.uint8).cuda()
        flat_ref = np.concatenate([g.cpu().numpy().ravel() for g in grads])
        for wire, dt in ((N.WIRE_F32, torch.float32), (N.WIRE_BF16, torch.bfloat16)):
            flat = torch.zeros(total, dtype=dt, device='cuda')
            N.check(lib.dmlb_multi_pack(dsegs.data_ptr(), len(grads), total, flat.data_ptr(), wire, 0.25, sptr()))
            want = grad_oracle.scale_f32(flat_ref, 4)
            if wire == N.WIRE_BF16:
                want = grad_oracle.round_bf16(want)
            assert (flat.float().cpu().numpy() == want).all()
            outs = [torch.zeros_like(g) for g in grads]
            for i, o in enumerate(outs):
                segs[i].ptr = o.data_ptr()
            dsegs2 = torch.frombuffer(bytearray(bytes(segs)), dtype=torch.uint8).cuda()
            sumsq = torch.zeros(1, dtype=torch.float64, device='cuda')
            N.check(lib.dmlb_multi_unpack(dsegs2.data_ptr(), len(grads), total, flat.data_ptr(), wire, 1.0,
                                          sumsq.data_ptr(), sptr()))
            got = np.concatenate([o.cpu().numpy().ravel() for o in outs])
            assert (got == want).all()
            np.testing.assert_allclose(sumsq.item(), np.sum(want.astype(np.float64) ** 2), rtol=1e-12)

    def test_roundtrip_property_at_full_size(self, lib):
        """ResNet-18-sized bucket (11,689,512 fp32): pack->unpack is idempotent and linear in the scale (size-
        independent properties; the oracle is only run on a strided sample)."""
        n = 11_689_512
        g = torch.randn(n, device='cuda')
        wire = torch.empty(n, dtype=torch.bfloat16, device='cuda')
        out1, out2 = torch.empty_like(g), torch.empty_like(g)
        N = N_()
        N.check(lib.dmlb_bucket_pack_f32_bf16(g.data_ptr(), wire.data_ptr(), n, 0.125, sptr()))
        N.check(lib.dmlb_bucket_unpack_bf16_f32(wire.data_ptr(), out1.data_ptr(), n, 1.0, None, sptr()))
        N.check(lib.dmlb_bucket_pack_f32_bf16(out1.data_ptr(), wire.data_ptr(), n, 1.0, sptr()))
        N.check(lib.dmlb_bucket_unpack_bf16_f32(wire.data_ptr(), out2.data_ptr(), n, 1.0, None, sptr()))
        assert torch.equal(out1, out2)  # bf16 values are fixed points of the cast
        assert torch.equal(out1, (g * 0.125).to(torch.bfloat16).float())
        idx = np.arange(0, n, 9973)
        want = grad_oracle.round_bf16(grad_oracle.scale_f32(g.cpu().numpy()[idx], 8))
        assert (out1.cpu().numpy()[idx] == want).all()


def _sms():
    return N_().device_info(0)['sm_count']


STREAM_ENTRIES = ['scale', 'pack_f32', 'pack_bf16', 'unpack_bf16_sumsq', 'round_bf16_sumsq', 'sumsq', 'clip']
STREAM_FUNCTOR = {'scale': 'ScaleInplace', 'pack_f32': 'PackF32', 'pack_bf16': 'PackBf16',
                  'unpack_bf16_sumsq': 'UnpackBf16<true>', 'round_bf16_sumsq': 'RoundBf16Inplace<true>',
                  'sumsq': 'SumsqF32', 'clip': 'ClipF32'}
STREAM_REGIMES = ['last_first_wave', 'first_rounded_grid', 'last_chunked', 'first_grid_stride', 'grid_stride_head']


def _f64_sumsq(x):
    return float(np.sum(np.asarray(x, dtype=np.float64) ** 2))


def _run_stream_entry(lib, entry, n, off, seed):
    """One launch_stream entry point on n elements starting `off` elements into a 16-byte aligned allocation (so the
    kernel's scalar head is (4 - off) % 4 elements).  Returns (got, want, sumsq got, sumsq want, launches)."""
    from helpers import check_launches, dmlb_launches

    N = N_()
    g = rand_grads(n + 8, seed)
    gv = g[off:off + n]
    st = sptr()
    sumsq = torch.zeros(1, dtype=torch.float64, device='cuda')
    want_sq = None
    if entry in ('scale', 'round_bf16_sumsq', 'sumsq', 'clip'):
        x = torch.from_numpy(g).cuda()[off:off + n]
        if entry == 'scale':
            call = lambda: lib.dmlb_bucket_scale_f32(x.data_ptr(), n, 0.125, st)
            want = grad_oracle.scale_f32(gv, 8)
        elif entry == 'round_bf16_sumsq':
            call = lambda: lib.dmlb_bucket_round_bf16_f32(x.data_ptr(), n, 0.25, sumsq.data_ptr(), st)
            want = grad_oracle.round_bf16(grad_oracle.scale_f32(gv, 4))
            want_sq = _f64_sumsq(want)
        elif entry == 'sumsq':
            call = lambda: lib.dmlb_bucket_sumsq_f32(x.data_ptr(), n, sumsq.data_ptr(), st)
            want, want_sq = gv, _f64_sumsq(gv)
        else:  # clip: the coefficient is formed on the device from the fp64 sum, in fp32 like clip_grad_norm_
            sq = _f64_sumsq(gv)
            sumsq.fill_(sq)
            total = np.float32(np.sqrt(sq))
            coef = min(np.float32(1.0), np.float32(np.float32(1.5) / np.float32(total + np.float32(1e-6))))
            call = lambda: lib.dmlb_bucket_clip_f32(x.data_ptr(), n, sumsq.data_ptr(), 1.5, st)
            want = (gv * np.float32(coef)).astype(np.float32)
        out = x
    elif entry == 'pack_f32':
        x = torch.from_numpy(g).cuda()[off:off + n]
        out = torch.zeros(n + 8, device='cuda')[off:off + n]
        call = lambda: lib.dmlb_bucket_pack_f32_f32(x.data_ptr(), out.data_ptr(), n, 0.125, st)
        want = grad_oracle.scale_f32(gv, 8)
    elif entry == 'pack_bf16':
        x = torch.from_numpy(g).cuda()[off:off + n]
        wire = torch.zeros(n + 8, dtype=torch.bfloat16, device='cuda')
        out = wire[off:off + n]
        call = lambda: lib.dmlb_bucket_pack_f32_bf16(x.data_ptr(), out.data_ptr(), n, 0.125, st)
        want = grad_oracle.round_bf16(grad_oracle.scale_f32(gv, 8))
    else:  # unpack_bf16_sumsq
        bits = grad_oracle.f32_to_bf16_bits(g)
        src = torch.from_numpy(bits.view(np.int16)).cuda().view(torch.bfloat16)[off:off + n]
        out = torch.full((n + 8,), -7.0, device='cuda')[off:off + n]
        call = lambda: lib.dmlb_bucket_unpack_bf16_f32(src.data_ptr(), out.data_ptr(), n, 2.0, sumsq.data_ptr(), st)
        want = grad_oracle.bf16_bits_to_f32(bits[off:off + n]) * np.float32(2.0)
        want_sq = _f64_sumsq(want)
    rc, launches = dmlb_launches(call)
    N.check(rc, entry)
    got = out.float().cpu().numpy() if entry != 'sumsq' else gv
    return got, want, sumsq.item(), want_sq, launches


class TestBucketKernelBoundaries:
    """Every launch_stream entry point at the edges of its launch regimes on this device (tests/launch_geometry.py):
    the last one-CTA-per-SM grid, the first grid rounded up to a multiple of the SM count, the last two-wave chunked
    launch, the first grid-stride launch and a grid-stride launch with an unaligned scalar head."""

    @pytest.mark.parametrize('regime', STREAM_REGIMES)
    @pytest.mark.parametrize('entry', STREAM_ENTRIES)
    def test_stream_entry_at_regime_edge(self, lib, entry, regime):
        import launch_geometry as G
        from helpers import check_launches

        sms = _sms()
        sizes = G.stream_sizes(sms)
        if regime == 'grid_stride_head':
            n, off = sizes['first_grid_stride'] + 4097, 1 + STREAM_ENTRIES.index(entry) % 3
        else:
            n, off = sizes[regime], 0
        head = (4 - off) % 4
        grid, chunk = G.launch_stream(n, head, sms)
        assert (chunk == 0) == (regime in ('first_grid_stride', 'grid_stride_head'))
        got, want, sq, want_sq, launches = _run_stream_entry(lib, entry, n, off, 1000 + n + off)
        check_launches(launches, [(f'dmlb::stream_kernel<dmlb::{STREAM_FUNCTOR[entry]}, {"true" if want_sq else "false"}>',
                                   grid)])
        assert (got.view(np.uint32) == want.view(np.uint32)).all(), int((got != want).sum())
        if want_sq is not None:
            np.testing.assert_allclose(sq, want_sq, rtol=1e-12)

    @pytest.mark.parametrize('case', ['regs_below_tma', 'tma', 'tma_plus_tail', 'tma_size_misaligned'])
    def test_bf16_dispatcher_hands_over_to_tma(self, lib, case):
        """dmlb_bucket_pack_f32_bf16 / unpack_bf16_f32 take the TMA kernels from kTmaMinElems on when both pointers are
        16-byte aligned, the register kernels otherwise; a ragged tail after the TMA body is one more launch."""
        import launch_geometry as G
        from helpers import check_launches, dmlb_launches

        N = N_()
        n = {'regs_below_tma': G.K_TMA_MIN_ELEMS - 1, 'tma': G.K_TMA_MIN_ELEMS, 'tma_plus_tail': G.K_TMA_MIN_ELEMS + 5,
             'tma_size_misaligned': G.K_TMA_MIN_ELEMS}[case]
        off = 1 if case == 'tma_size_misaligned' else 0
        g = torch.randn(n + 8, device='cuda')
        src = g[off:off + n]
        wire = torch.zeros(n + 8, dtype=torch.bfloat16, device='cuda')[off:off + n]
        out = torch.full((n + 8,), -3.0, device='cuda')[off:off + n]
        st = sptr()

        def both():
            N.check(lib.dmlb_bucket_pack_f32_bf16(src.data_ptr(), wire.data_ptr(), n, 0.125, st))
            N.check(lib.dmlb_bucket_unpack_bf16_f32(wire.data_ptr(), out.data_ptr(), n, 2.0, None, st))

        _, launches = dmlb_launches(both)
        regs = ['dmlb::stream_kernel<dmlb::PackBf16, false>', 'dmlb::stream_kernel<dmlb::UnpackBf16<false>, false>']
        want_names = {'regs_below_tma': regs, 'tma_size_misaligned': regs,
                      'tma': ['dmlb::pack_bf16_tma_kernel', 'dmlb::unpack_bf16_tma_kernel'],
                      'tma_plus_tail': ['dmlb::pack_bf16_tma_kernel', regs[0], 'dmlb::unpack_bf16_tma_kernel', regs[1]]}
        if case in ('regs_below_tma', 'tma_size_misaligned'):  # the register path: grids as launch_stream picks them
            grid = G.launch_stream(n, (4 - off) % 4, _sms())[0]
            check_launches(launches, [(regs[0], grid), (regs[1], grid)])
        else:  # TMA: its grid is not restated; the kernel sequence is the witness
            check_launches(launches, [(k, g) for k, (_, g) in zip(want_names[case], launches)])
        gv = src.cpu().numpy()
        want = grad_oracle.round_bf16(grad_oracle.scale_f32(gv, 8))
        assert (wire.float().cpu().numpy() == want).all()
        assert (out.cpu().numpy() == want * np.float32(2.0)).all()


class TestShardKernels:
    def test_gather_normalise_matches_torchvision_arithmetic(self, lib):
        N = N_()
        rng = np.random.RandomState(0)
        images = torch.from_numpy(rng.randint(0, 256, (500, 1, 28, 28)).astype(np.uint8)).cuda()
        labels = torch.from_numpy(rng.randint(0, 10, 500)).cuda()
        idx = torch.from_numpy(rng.permutation(500)[:64]).cuda()
        x = torch.empty(64, 1, 28, 28, device='cuda')
        y = torch.empty(64, dtype=torch.int64, device='cuda')
        N.check(lib.dmlb_shard_gather_u8(images.data_ptr(), idx.data_ptr(), 64, 784, 0.1307, 0.3081, x.data_ptr(), 0,
                                         sptr()))
        N.check(lib.dmlb_shard_gather_i64(labels.data_ptr(), idx.data_ptr(), 64, y.data_ptr(), sptr()))
        # ToTensor: uint8 -> float / 255 ; Normalize: (x - mean) / std     (examples/mnist.py:16)
        want = (images[idx].cpu().float().div(255).sub(0.1307).div(0.3081))
        assert torch.equal(x.cpu(), want)
        assert torch.equal(y.cpu(), labels[idx].cpu())
        xb = torch.empty(64, 1, 28, 28, dtype=torch.bfloat16, device='cuda')
        N.check(lib.dmlb_shard_gather_u8(images.data_ptr(), idx.data_ptr(), 64, 784, 0.1307, 0.3081, xb.data_ptr(), 1,
                                         sptr()))
        assert torch.equal(xb.cpu(), want.to(torch.bfloat16))
        # ragged row size -> scalar path
        odd = images.reshape(500, 784)[:, :781].contiguous()
        xo = torch.empty(64, 781, device='cuda')
        N.check(lib.dmlb_shard_gather_u8(odd.data_ptr(), idx.data_ptr(), 64, 781, 0.5, 2.0, xo.data_ptr(), 0, sptr()))
        assert torch.equal(xo.cpu(), odd[idx].cpu().float().div(255).sub(0.5).div(2.0))

    def test_device_sharded_dataset_is_bit_exact_with_reference_indices(self):
        from dmlcloud_b200.util.data import DeviceShardedDataset
        from oracle import shard

        rng = np.random.RandomState(1)
        n = 1003
        images = torch.from_numpy(rng.randint(0, 256, (n, 1, 28, 28)).astype(np.uint8))
        labels = torch.arange(n)  # label == dataset index, so the batches reveal the indices
        seen = {}
        for rank in range(4):
            ds = DeviceShardedDataset(images, labels, batch_size=32, shuffle=True, seed=7, rank=rank, world_size=4,
                                      device='cuda:0')
            ds.set_epoch(3)
            got = torch.cat([y for _, y in ds]).cpu().tolist()
            assert got == shard.shard_indices(n, rank, 4, True, True, 7 + 3)  # seed + epoch, util/data.py:139-146
            assert len(ds) == -(-len(got) // 32)
            seen[rank] = got
            x0, y0 = next(iter(ds))
            assert torch.equal(x0.cpu(), images[y0.cpu()].float().div(255).sub(0.1307).div(0.3081))
        flat = sum(seen.values(), [])
        assert len(set(flat)) == len(flat) == n - n % 4
        gold = load_json('shard_indices.json')
        case = next(c for c in gold['cases'] if c['n'] == 1000 and c['shuffle'] and c['even_shards'] and c['rank'] == 2)
        ds = DeviceShardedDataset(images[:1000], labels[:1000], batch_size=50, shuffle=True, seed=case['seed'],
                                  rank=2, world_size=case['world'], device='cuda:0')
        assert torch.cat([y for _, y in ds]).cpu().tolist() == case['out']  # epoch 0 -> the reference's own list

    @pytest.mark.parametrize('out_bf16', [0, 1], ids=['fp32', 'bf16'])
    def test_gather_at_capped_grid(self, lib, out_bf16):
        """A batch of 8,192 MNIST images: more 16-pixel vectors than the grid (capped at 8 CTAs per SM) has threads, so
        every thread walks several of them."""
        import launch_geometry as G
        from helpers import check_launches, dmlb_launches

        N = N_()
        batch, row = 8192, 784
        rng = np.random.RandomState(4)
        images = torch.from_numpy(rng.randint(0, 256, (10000, row)).astype(np.uint8)).cuda()
        idx = torch.from_numpy(rng.randint(0, 10000, batch)).cuda()
        dt = torch.bfloat16 if out_bf16 else torch.float32
        x = torch.empty(batch, row, dtype=dt, device='cuda')
        rc, launches = dmlb_launches(lambda: lib.dmlb_shard_gather_u8(images.data_ptr(), idx.data_ptr(), batch, row, 0.1307,
                                                                      0.3081, x.data_ptr(), out_bf16, sptr()))
        N.check(rc)
        grid = G.shard_grid(batch * row // 16, _sms())
        check_launches(launches, [(f'dmlb::shard_gather_u8_kernel<{"true" if out_bf16 else "false"}>', grid)])
        assert grid * 256 < batch * row // 16
        want = images[idx].cpu().float().div(255).sub(0.1307).div(0.3081)
        assert torch.equal(x.cpu(), want.to(dt))
