"""CPU: the C-ABI shared library loads and exports every symbol include/b200_e2tts.h declares (no compute calls)."""
import ctypes
import os
import subprocess

import pytest

from conftest import ROOT


@pytest.fixture(scope='module')
def pkg():
    so = os.path.join(ROOT, 'e2-tts-pytorch_b200', 'libb200e2tts.so')
    if not os.path.isfile(so):
        subprocess.run(['make', '-C', os.path.join(ROOT, 'e2-tts-pytorch_b200', 'csrc'), '-j8', 'all'], check=True)
    import e2_tts_pytorch_b200 as pkg
    return pkg


def test_every_declared_symbol_is_exported(pkg):
    lib = pkg.lib.load()
    assert len(pkg.lib.FUNCTIONS) >= 30
    for name in pkg.lib.FUNCTIONS:
        assert hasattr(lib, name), name
    assert lib.b200_version() == 90   # built for sm_90a
    assert isinstance(pkg.lib.launch_count(), int)


def test_struct_layouts_parse(pkg):
    for name, fields in pkg.lib.STRUCT_FIELDS.items():
        assert fields, name
        assert ctypes.sizeof(pkg.lib.STRUCTS[name]) > 0
    # spot check: the GEMM descriptor of the header has the documented leading fields
    assert [f for f, _ in pkg.lib.STRUCT_FIELDS['b200_gemm_args']][:5] == ['A', 'lda', 'A2', 'lda2', 'K1']


def test_argument_validation_without_gpu(pkg):
    """Entry points reject bad arguments before touching the device (error string through b200_last_error)."""
    a = pkg.lib.make_args('b200_gemm_args', M=0, N=0, K=0)
    with pytest.raises(RuntimeError, match='gemm'):
        pkg.lib.call('b200_gemm', a, None)
    a = pkg.lib.make_args('b200_hc_width_args', num_streams=3)
    with pytest.raises(RuntimeError):
        pkg.lib.call('b200_hc_width_fwd', a, None)
    # the wgmma attention exponentiates without a running maximum: a softclamp above 64 is refused (placeholder pointers, never read)
    ptrs = dict.fromkeys(('q', 'k', 'v', 'o', 'lse', 'ws_maskbits'), 256)
    shape = dict(B=1, H=1, Np=64, dim_head=64, scale=0.125, softclamp=100.0)
    a = pkg.lib.make_args('b200_attn_fwd_args', og=256, **ptrs, **shape)
    with pytest.raises(RuntimeError, match='softclamp'):
        pkg.lib.call('b200_attn_fwd', a, None)
    a = pkg.lib.make_args('b200_attn_bwd_args', d_og=256, ws_dO=256, ws_delta=256, dq=256, dk=256, dv=256, **ptrs, **shape)
    with pytest.raises(RuntimeError, match='softclamp'):
        pkg.lib.call('b200_attn_bwd', a, None)


def test_state_dict_is_reference_compatible(pkg):
    import torch
    g = torch.load(os.path.join(ROOT, 'tests', 'golden', 'e2tts_d128_L2.pt'), weights_only=False)
    m = pkg.E2TTS(transformer=dict(dropout=0., max_seq_len=g['max_seq_len'], **g['transformer']), use_vocos=False)
    assert set(m.state_dict().keys()) == set(g['state_dict'].keys())
    m.load_state_dict(g['state_dict'])
    d = torch.load(os.path.join(ROOT, 'tests', 'golden', 'duration_d128_L2.pt'), weights_only=False)
    dp = pkg.DurationPredictor(transformer=dict(dropout=0., max_seq_len=256, **g['transformer']))
    assert set(dp.state_dict().keys()) == set(d['state_dict'].keys())


def test_unsupported_switches_raise(pkg):
    with pytest.raises(NotImplementedError):
        pkg.Transformer(dim=128, depth=2, heads=2, attn_laser=True)
    with pytest.raises(NotImplementedError):
        pkg.Transformer(dim=128, depth=2, heads=2, has_freq_axis=True)
    with pytest.raises(NotImplementedError):
        pkg.E2TTS(transformer=dict(dim=128, depth=2, heads=2), num_freq_tokens=2, use_vocos=False)
    # the variants that ARE built construct with the reference's parameter layout (SURVEY §8f row 4)
    m = pkg.E2TTS(transformer=dict(dim=128, depth=2, heads=2, attn_fourier_embed_input=True), concat_cond=True, interpolated_text=True, use_vocos=False)
    sd = m.state_dict()
    assert sd['proj_in.weight'].shape == (128, 200) and 'cond_proj_in.weight' not in sd
    assert sd['embed_text.abs_pos_mlp.3.weight'].shape == (64, 64) and sd['transformer.layers.0.0.4.linear.weight'].shape == (96, 128)


def test_tokenizer_and_mask_helpers(pkg):
    import torch
    ids = pkg.list_str_to_tensor(['Hello', 'Goodbye'])
    assert ids.tolist() == [[72, 101, 108, 108, 111, -1, -1], [71, 111, 111, 100, 98, 121, 101]]
    assert pkg.lens_to_mask(torch.tensor([2, 3]), 3).tolist() == [[True, True, False], [True, True, True]]
    m = pkg.mask_from_frac_lengths(torch.tensor([10, 6]), torch.tensor([0.7, 1.0]), 10)
    assert m.sum(-1).tolist() == [7, 6] and not m[1, 6:].any()


def test_graphed_train_step_validates_its_arguments(pkg):
    """GraphedTrainStep (CUDA-graph replay of forward + backward) refuses what it cannot capture — checked without a GPU."""
    import pytest
    import torch
    m = pkg.E2TTS(transformer=dict(dim=128, depth=2, heads=2), use_vocos=False)
    m.cond_drop_prob = 0.0
    with pytest.raises(ValueError, match='GPU'):
        pkg.GraphedTrainStep(m, torch.randn(2, 32, 100))
    m.cond_drop_prob = 0.25   # the text-drop coin is a host-side branch: it would be frozen into the graph
    with pytest.raises(ValueError, match='cond_drop_prob'):
        pkg.GraphedTrainStep(m, torch.randn(2, 32, 100))


def test_positional_struct_marshalling_checks_the_header_order(pkg):
    """ops.gemm fills b200_gemm_args positionally (hot path): the binding verifies the order against the parsed header."""
    import pytest
    from e2_tts_pytorch_b200 import lib, ops
    declared = [f for f, _ in lib.STRUCT_FIELDS['b200_gemm_args']]
    assert tuple(declared[:len(ops._GEMM_FIELDS)]) == ops._GEMM_FIELDS
    s = lib.make_args_positional('b200_gemm_args', ops._GEMM_FIELDS, [None, 8] + [0] * (len(ops._GEMM_FIELDS) - 2))
    assert s.lda == 8 and s.force_tile == 0
    with pytest.raises(RuntimeError, match='field order'):
        lib.make_args_positional('b200_gemm_args', ('lda', 'A'), (8, None))


def test_host_helpers_of_the_round2_paths(pkg):
    """Host-side pieces of the fused hyper-connection path and of InterpolatedCharacterEmbed (no kernel calls)."""
    import torch
    from e2_tts_pytorch_b200 import ops
    assert ops.hc_can_fuse(16 * 1056, 4) and ops.hc_can_fuse(2 * 1312, 4) and not ops.hc_can_fuse(2 * 150, 4)
    text = torch.tensor([[5, -1, 7, 9, -1], [-1, -1, -1, -1, -1], [1, 2, 3, 4, 5]])
    ids, n = pkg.modules.InterpolatedCharacterEmbed.compact(text)
    assert n.tolist() == [3, 0, 5] and ids.dtype == torch.int32
    assert ids[0, :3].tolist() == [5, 7, 9] and ids[2].tolist() == [1, 2, 3, 4, 5]
