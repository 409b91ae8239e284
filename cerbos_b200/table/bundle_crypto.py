"""Encrypted rule-table bundles (`*.crrts`): the stream cipher layer in front of the serialized runtimev1.RuleTable.

The reference decrypts with ``crypto.DecryptChaCha20Poly1305Stream(key, in, out)`` (internal/storage/hub/
ruletable_bundle.go:56-70) from github.com/cerbos/cloud-api -- a third-party module outside the reference tree.  The
format restated here was identified on the reference's own fixture (internal/test/testdata/bundle/v2_ruletable/
bundle.crrts + encryption_key.txt, 48 bytes longer than its 131 518-byte plaintext) and is pinned by it: the STREAM
construction over ChaCha20-Poly1305 (RFC 8439) --

    plaintext in chunks of 64 KiB, every chunk sealed on its own (16-byte tag appended),
    nonce of chunk i = 11-byte big-endian counter i || 1 byte: 0x01 on the last chunk, else 0x00,
    no header, no associated data; the key is the 32-byte bundle key

-- every chunk authenticates, and the decrypted message decodes to the same 126 rule rows as bundle_unencrypted.crrt
(tests/test_ruletable_bundle.py).  ChaCha20 and Poly1305 are written out below (RFC 8439 §2.3, §2.5, §2.8); when the
`cryptography` package is importable its AEAD is used instead (same result, faster).
"""
from __future__ import annotations

import struct

CHUNK = 64 * 1024
TAG = 16


class BundleCryptoError(ValueError):
    pass


def _rotl(v, c):
    return ((v << c) & 0xFFFFFFFF) | (v >> (32 - c))


def _chacha20_block(key_words, counter, nonce_words):
    s = [0x61707865, 0x3320646E, 0x79622D32, 0x6B206574] + key_words + [counter] + nonce_words
    x = list(s)

    def qr(a, b, c, d):
        x[a] = (x[a] + x[b]) & 0xFFFFFFFF; x[d] = _rotl(x[d] ^ x[a], 16)
        x[c] = (x[c] + x[d]) & 0xFFFFFFFF; x[b] = _rotl(x[b] ^ x[c], 12)
        x[a] = (x[a] + x[b]) & 0xFFFFFFFF; x[d] = _rotl(x[d] ^ x[a], 8)
        x[c] = (x[c] + x[d]) & 0xFFFFFFFF; x[b] = _rotl(x[b] ^ x[c], 7)

    for _ in range(10):
        qr(0, 4, 8, 12); qr(1, 5, 9, 13); qr(2, 6, 10, 14); qr(3, 7, 11, 15)
        qr(0, 5, 10, 15); qr(1, 6, 11, 12); qr(2, 7, 8, 13); qr(3, 4, 9, 14)
    return struct.pack("<16I", *[(a + b) & 0xFFFFFFFF for a, b in zip(x, s)])


def _chacha20_xor(key: bytes, nonce: bytes, counter: int, data: bytes) -> bytes:
    kw = list(struct.unpack("<8I", key))
    nw = list(struct.unpack("<3I", nonce))
    out = bytearray()
    for off in range(0, len(data), 64):
        ks = _chacha20_block(kw, counter + off // 64, nw)
        blk = data[off:off + 64]
        out += bytes(a ^ b for a, b in zip(blk, ks))
    return bytes(out)


def _poly1305(key32: bytes, msg: bytes) -> bytes:
    r = int.from_bytes(key32[:16], "little") & 0x0FFFFFFC0FFFFFFC0FFFFFFC0FFFFFFF
    s = int.from_bytes(key32[16:], "little")
    p = (1 << 130) - 5
    acc = 0
    for off in range(0, len(msg), 16):
        blk = msg[off:off + 16]
        acc = ((acc + int.from_bytes(blk + b"\x01", "little")) * r) % p
    return ((acc + s) & ((1 << 128) - 1)).to_bytes(16, "little")


def _pad16(b: bytes) -> bytes:
    return b"\0" * (-len(b) % 16)


def open_chacha20poly1305(key: bytes, nonce: bytes, sealed: bytes, aad: bytes = b"") -> bytes:
    """RFC 8439 §2.8 AEAD open: sealed = ciphertext || 16-byte tag.  Raises BundleCryptoError if the tag does not verify."""
    if len(key) != 32 or len(nonce) != 12 or len(sealed) < TAG:
        raise BundleCryptoError("bad key / nonce / ciphertext length")
    ct, tag = sealed[:-TAG], sealed[-TAG:]
    otk = _chacha20_block(list(struct.unpack("<8I", key)), 0, list(struct.unpack("<3I", nonce)))[:32]
    mac = _poly1305(otk, aad + _pad16(aad) + ct + _pad16(ct) + struct.pack("<QQ", len(aad), len(ct)))
    diff = 0
    for a, b in zip(mac, tag):
        diff |= a ^ b
    if diff:
        raise BundleCryptoError("authentication failed (wrong key, or not an encrypted rule-table bundle)")
    return _chacha20_xor(key, nonce, 1, ct)


def _open(key: bytes, nonce: bytes, sealed: bytes) -> bytes:
    try:
        from cryptography.exceptions import InvalidTag
        from cryptography.hazmat.primitives.ciphers.aead import ChaCha20Poly1305
    except Exception:  # noqa: BLE001 -- not installed: the implementation above
        return open_chacha20poly1305(key, nonce, sealed)
    try:
        return ChaCha20Poly1305(key).decrypt(nonce, sealed, None)
    except InvalidTag as e:
        raise BundleCryptoError("authentication failed (wrong key, or not an encrypted rule-table bundle)") from e


def parse_key(key) -> bytes:
    """32 raw bytes, or their 64 hex digits (the form of the reference's encryption_key.txt)"""
    if isinstance(key, str):
        key = key.strip().encode("ascii")
    if len(key) == 64:
        try:
            key = bytes.fromhex(key.decode("ascii"))
        except ValueError as e:
            raise BundleCryptoError("bundle key: 64 characters that are not hex digits") from e
    if len(key) != 32:
        raise BundleCryptoError(f"bundle key must be 32 bytes (or 64 hex digits), got {len(key)}")
    return bytes(key)


def decrypt_stream(key, data: bytes) -> bytes:
    """crypto.DecryptChaCha20Poly1305Stream: -> the serialized runtimev1.RuleTable"""
    key = parse_key(key)
    data = bytes(data)
    if len(data) < TAG:
        raise BundleCryptoError("encrypted bundle too short")
    out = bytearray()
    n_chunks = (len(data) + CHUNK + TAG - 1) // (CHUNK + TAG)
    for i in range(n_chunks):
        sealed = data[i * (CHUNK + TAG):(i + 1) * (CHUNK + TAG)]
        last = i == n_chunks - 1
        if len(sealed) < TAG or (not last and len(sealed) != CHUNK + TAG):
            raise BundleCryptoError("encrypted bundle truncated")
        nonce = i.to_bytes(11, "big") + (b"\x01" if last else b"\x00")
        out += _open(key, nonce, sealed)
    return bytes(out)
