"""``BitPack`` with the reference's API (hqq/core/bitpack.py:10-144), executed by the sm_90a library.

Layout is bit-identical to the reference ("slab interleave" along dim 0, most significant field
first; 3-bit = 10 fields per int32 with zero-padded rows); see tests/test_bitpack.py.
"""
from __future__ import annotations

import torch
from torch import Tensor, uint8

from .. import ops


class BitPack:
    # 8-bit ------------------------------------------------------------------
    @staticmethod
    def pack_8bit_u8(W_q: Tensor) -> Tensor:
        return ops.pack(W_q, 8)

    @staticmethod
    def unpack_8bit_u8(W_q: Tensor, dtype=uint8) -> Tensor:
        return ops.unpack(W_q, 8, dtype)

    # 4-bit ------------------------------------------------------------------
    @staticmethod
    def pack_4bit_u8(W_q: Tensor) -> Tensor:  # [R, C] -> uint8 [R/2, C]
        return ops.pack(W_q, 4)

    @staticmethod
    def unpack_4bit_u8(W_q: Tensor, dtype=uint8) -> Tensor:  # uint8 [R/2, C] -> [R, C]
        return ops.unpack(W_q, 4, dtype)

    # 2-bit ------------------------------------------------------------------
    @staticmethod
    def pack_2bit_u8(W_q: Tensor) -> Tensor:
        return ops.pack(W_q, 2)

    @staticmethod
    def unpack_2bit_u8(W_q: Tensor, dtype=uint8) -> Tensor:
        return ops.unpack(W_q, 2, dtype)

    # 3-bit ------------------------------------------------------------------
    @staticmethod
    def pack_3bit_32(W_q_in: Tensor) -> Tensor:  # [R, C] -> int32 [ceil(R/10), C]
        return ops.pack(W_q_in, 3)

    @staticmethod
    def unpack_3bit_32(W_q: Tensor, dtype=uint8) -> Tensor:  # keeps the padded rows, like the reference
        return ops.unpack(W_q, 3, dtype)

    # 1-bit ------------------------------------------------------------------
    @staticmethod
    def pack_1bit_u8(W_q: Tensor) -> Tensor:
        return ops.pack(W_q, 1)

    @staticmethod
    def unpack_1bit_u8(W_q: Tensor, dtype=uint8) -> Tensor:
        return ops.unpack(W_q, 1, dtype)
