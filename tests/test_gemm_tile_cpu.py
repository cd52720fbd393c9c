"""The GEMM's output-tile width rule (pulse_gemm_tile_n) on the update's shapes, for an H100's 132 SMs: no GPU needed."""
import pytest


@pytest.fixture(scope="module")
def lib():
    from pulse_b200 import build
    build.build()
    from pulse_b200 import _lib
    return _lib.load()


# (M, N, K, expected width): forward and input-gradient GEMMs of one PPO + discriminator minibatch
SHAPES = [
    (16384, 1024, 960, 256),    # actor / critic layer 1 forward
    (16384, 512, 1024, 256),    # actor / critic layer 2 forward
    (16384, 69, 512, 128),      # actor head: 69 columns
    (16384, 512, 69, 128),      # actor head dgrad: 2 k-blocks per item
    (16384, 1024, 512, 256),    # actor / critic layer 2 dgrad
    (12288, 1024, 1984, 256),   # discriminator layer 1 forward
    (12288, 512, 1024, 128),    # discriminator layer 2 forward: 192 wide items take 2 rounds, 384 narrow ones 3
    (12288, 1024, 512, 256),    # discriminator layer 2 dgrad
    (4096, 1024, 512, 256),     # gradient penalty g1
    (4096, 1960, 1024, 256),    # gradient penalty G
    (4096, 1024, 1960, 256),    # gradient penalty du
]


@pytest.mark.parametrize("M,N,K,width", SHAPES)
def test_update_shapes(lib, M, N, K, width):
    assert lib.pulse_gemm_tile_n(M, N, K, 1, 132) == width


def test_wide_needs_a_round_saved(lib):
    # 64 narrow items fit one round on 132 SMs; 32 wide ones would leave half the SMs idle for the same round
    assert lib.pulse_gemm_tile_n(4096, 256, 1088, 1, 132) == 128
    # fewer SMs: the same shape takes 2 narrow rounds against 1 wide one
    assert lib.pulse_gemm_tile_n(4096, 256, 1088, 1, 32) == 256
