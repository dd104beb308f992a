"""One wire packet per session per transmitter step: a fixed 16-byte little-endian header and the packed code frames.

    offset  size  field
    0       2     magic, the ASCII bytes "AD" (0x41 0x44)
    2       1     version, 1
    3       1     codebook_num: code indices per frame (Nq)
    4       4     session id, u32
    8       4     sequence number, u32: 0 for a session's first packet, one more for each packet after it
    12      2     frames: code frames in the payload, u16, at least 1
    14      2     frame_bytes: packed bytes per frame, u16
    16      ...   payload: frames x frame_bytes bytes, frame after frame

Each payload frame is the packed bitstream the fused RVQ writes (``quantize_fused(want_packed=True)``, ``adec_quantize_ex``;
DESIGN.md §4.4): Nq local indices of ceil(log2 codebook_size) bits, stage 0 first, little-endian bit order, zero-padded to whole
bytes.  ``lookup_packed`` reads it back.  The buffer a receiver gets comes from outside the program, so ``decode_packet`` checks
every header field against the buffer and the receiver's codec before anything reaches the GPU.
"""
from __future__ import annotations

import struct
from typing import NamedTuple, Optional

MAGIC = b"AD"
VERSION = 1
_HEADER = struct.Struct("<2sBBIIHH")
HEADER_BYTES = _HEADER.size          # 16


class Packet(NamedTuple):
    session_id: int
    seq: int
    frames: int
    codebook_num: int
    frame_bytes: int
    payload: bytes


def encode_packet(session_id: int, seq: int, codebook_num: int, frame_bytes: int, payload) -> bytes:
    """The packet of `payload` (bytes-like, a whole number of `frame_bytes`-byte packed frames) for session `session_id`."""
    payload = bytes(payload)
    if not 0 <= session_id < 1 << 32:
        raise ValueError(f"session_id {session_id} does not fit in a u32")
    if not 0 <= seq < 1 << 32:
        raise ValueError(f"seq {seq} does not fit in a u32")
    if not 1 <= codebook_num < 1 << 8:
        raise ValueError(f"codebook_num {codebook_num} does not fit in a u8")
    if not 1 <= frame_bytes < 1 << 16:
        raise ValueError(f"frame_bytes {frame_bytes} does not fit in a u16")
    frames, rest = divmod(len(payload), frame_bytes)
    if rest or not 1 <= frames < 1 << 16:
        raise ValueError(f"payload of {len(payload)} bytes is not 1 to 65535 frames of {frame_bytes} bytes")
    return _HEADER.pack(MAGIC, VERSION, codebook_num, session_id, seq, frames, frame_bytes) + payload


def decode_packet(buf, codebook_num: Optional[int] = None, frame_bytes: Optional[int] = None) -> Packet:
    """Parse and check one packet.  `codebook_num` / `frame_bytes`: what the receiver's codec expects (None: not checked).  Raises
    ValueError naming the field for a short header, a bad magic or version, a frame count of 0, a payload length other than
    frames x frame_bytes, or a codebook count or frame size other than the receiver's."""
    buf = bytes(buf)
    if len(buf) < HEADER_BYTES:
        raise ValueError(f"header: packet of {len(buf)} bytes is shorter than the {HEADER_BYTES}-byte header")
    magic, version, nq, session_id, seq, frames, nb = _HEADER.unpack_from(buf)
    if magic != MAGIC:
        raise ValueError(f"magic: expected {MAGIC!r}, got {magic!r}")
    if version != VERSION:
        raise ValueError(f"version: expected {VERSION}, got {version}")
    if codebook_num is not None and nq != codebook_num:
        raise ValueError(f"codebook_num: packet has {nq}, the receiver's codec {codebook_num}")
    if frame_bytes is not None and nb != frame_bytes:
        raise ValueError(f"frame_bytes: packet has {nb}, the receiver's codec {frame_bytes}")
    if frames == 0 or nb == 0:
        raise ValueError(f"frames: packet holds {frames} frames of {nb} bytes; a packet holds at least one frame of at least one byte")
    if len(buf) - HEADER_BYTES != frames * nb:
        raise ValueError(f"payload: {len(buf) - HEADER_BYTES} bytes, the header says {frames} frames x {nb} bytes = {frames * nb}")
    return Packet(session_id, seq, frames, nq, nb, buf[HEADER_BYTES:])
