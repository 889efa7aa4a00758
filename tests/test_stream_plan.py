"""tools/stream_bench.py's planning arithmetic for streamed layers, against values worked out by hand (no GPU).

A Q4_K block of 256 weights has three device planes of 128, 16 and 4 bytes (quants, expanded scales + mins, d + dmin).  A plane's rows
are padded to 16 bytes and the plane to 256 bytes (wplanes_layout).
"""
import importlib.util
import os

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def sb():
    spec = importlib.util.spec_from_file_location("stream_bench", os.path.join(ROOT, "tools", "stream_bench.py"))
    m = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(m)
    return m


def test_falcon_40b_q4_k_layer_image(sb):
    # n_embd 8192 = 32 blocks: rows of 4096 + 512 + 128 = 4736 bytes, none padded; ffn_down (K = 32768, 128 blocks): 16384 + 2048 + 512
    # qkv 9216 rows, wo 8192, ffn_up 32768, ffn_down 8192
    assert sb.matrix_image_bytes(sb.Q4_K, 8192, 9216) == 4736 * 9216 == 43646976
    assert sb.matrix_image_bytes(sb.Q4_K, 32768, 8192) == 18944 * 8192 == 155189248
    assert sb.layer_image_bytes(sb.FALCON_40B, sb.Q4_K) == 43646976 + 38797312 + 155189248 + 155189248 == 392822784


def test_falcon_180b_q4_k_layer_image(sb):
    # n_embd 14848 = 58 blocks: plane rows 7424, 928 and 232 -> 240 (16-byte padding); ffn_down 232 blocks: 29696, 3712, 928
    assert sb.matrix_image_bytes(sb.Q4_K, 14848, 15872) == (7424 + 928 + 240) * 15872 == 136372224
    assert sb.matrix_image_bytes(sb.Q4_K, 14848, 14848) == 127574016
    assert sb.matrix_image_bytes(sb.Q4_K, 59392, 14848) == (29696 + 3712 + 928) * 14848 == 509820928
    assert sb.layer_image_bytes(sb.FALCON_180B, sb.Q4_K) == 136372224 + 127574016 + 4 * 127574016 + 509820928 == 1284063232


def test_plane_padding_to_256_bytes(sb):
    # Q4_0, K = 64: rows of 2 x 16 quant bytes and 2 x 2 scale bytes -> 4 -> 16; 3 rows: 96 -> 256 and 48 -> 256
    assert sb.matrix_image_bytes(sb.Q4_0, 64, 3) == 512


def test_falcon_180b_resident_layers(sb):
    # embedding table + lm_head: 2 x 8592 x 65024; f32 KV cache at n_ctx 8192: 80 x 2 x 8192 x 512 x 4; activations for one token:
    # 4 x (5 x 14848 + 15872 + 59392 + 65024); two slots; 2 GiB margin
    fixed = 2 * 558686208 + 2684354560 + 858112 + 2 * 1284063232 + 2 * (1 << 30)
    assert fixed == 8518195200
    assert sb.plan_resident_layers(sb.FALCON_180B, sb.Q4_K, 84_000_000_000, 8192) == (84_000_000_000 - fixed) // 1284063232 == 58
    # a card that other jobs have partly filled keeps fewer layers; one with room for everything keeps all 80
    assert sb.plan_resident_layers(sb.FALCON_180B, sb.Q4_K, 40_000_000_000, 8192) == (40_000_000_000 - fixed) // 1284063232 == 24
    assert sb.plan_resident_layers(sb.FALCON_180B, sb.Q4_K, 200_000_000_000, 8192) == 80
    assert sb.plan_resident_layers(sb.FALCON_180B, sb.Q4_K, 1_000_000_000, 8192) == 0


def test_falcon_40b_resident_layers(sb):
    # n_ctx 2048, one token: 2 x 4736 x 65024 + 60 x 2 x 2048 x 512 x 4 + 4 x (5 x 8192 + 9216 + 32768 + 65024) + 2 layers + 2 GiB
    fixed = 2 * 307953664 + 503316480 + 591872 + 2 * 392822784 + 2 * (1 << 30)
    assert sb.plan_resident_layers(sb.FALCON_40B, sb.Q4_K, 20_000_000_000, 2048) == (20_000_000_000 - fixed) // 392822784 == 40
    # a prompt engine (512 tokens) also holds the fp16 K and V^T planes: 2 x 60 x 8 x 64 x 2048 x 2 bytes, and 512 activation rows
    fixed512 = fixed - 591872 + 512 * 591872 + 2 * 60 * 8 * 64 * 2048 * 2
    assert sb.plan_resident_layers(sb.FALCON_40B, sb.Q4_K, 20_000_000_000, 2048, n_batch=512) == (20_000_000_000 - fixed512) // 392822784
