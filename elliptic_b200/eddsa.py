"""Host-side mirror of the reference's EdDSA object for the accelerated path.

`EDDSA('ed25519')` corresponds to `new elliptic.eddsa('ed25519')`
(lib/elliptic/eddsa/index.js:11-25); `verify(message, sig, pub)` keeps the reference's
argument forms and error behaviour (eddsa/index.js:52-63) and `verify_batch` is the new
batch entry point.  Byte/hex parsing and the SHA-512 of R || A || M are done here
(hashlib; the reference uses hash.js); all curve arithmetic runs on the GPU.
"""
import ctypes
import hashlib

import numpy as np

from . import _native as nat
from .ec import EllipticError, _NativeSets, _answer, _blob, _pack, _to_array

N_ED25519 = 0x1000000000000000000000000000000014DEF9DEA2F79CD65812631A5CF5D3ED


def _parse_bytes(x):
    """utils.parseBytes (lib/elliptic/utils.js:112-116)."""
    return _to_array(x, "hex") if isinstance(x, str) else _to_array(x)


class _EdKeyObjects:
    """The key-object side of the `eddsa` API (eddsa/key.js), in batch form; EDDSA inherits it."""

    def key_set(self, pubs, table_bits=0):
        """The batch form of `key = eddsa.keyFromPublic(pub)` for many keys: an EdKeySet on the GPU."""
        return EdKeySet(self, pubs, table_bits)

    def signing_set(self, secrets):
        """The batch form of `key = eddsa.keyFromSecret(secret)` for many keys: an EdSigningSet on the GPU."""
        return EdSigningSet(self, secrets)


class _EdTensorForms:
    """The EdDSA device-buffer calls on CUDA tensors, on the caller's stream (conventions: _tensors); EDDSA inherits
    them."""

    def verify_batch_tensors(self, R, S, A, h):
        """verify_batch_packed on CUDA tensors (eb200_eddsa_verify_batch_dev): R, S, A, h (n, 32).  Returns the statuses."""
        from . import _tensors as T
        n, dev = T.check("verify_batch_tensors", [(a, t, T.ROWS, 32) for a, t in (("R", R), ("S", S), ("A", A), ("h", h))])
        st = T.empty(dev, n)
        T.launch("eb200_eddsa_verify_batch_dev", dev, [n, R, S, A, h, st], T.ws_unkeyed(nat.CURVE_ED25519, n))
        return st

    def verify_batch_msgs_tensors(self, R, S, A, msgs, msg_off):
        """verify_batch_msgs_packed on CUDA tensors (eb200_eddsa_verify_batch_msgs_dev): R, S, A (n, 32), the messages
        back to back in msgs (1-D uint8) with (n + 1,) int64 offsets.  Returns the statuses (ST_BAD_ITEM for a range that
        decreases or ends past msgs)."""
        from . import _tensors as T
        n, dev = T.check("verify_batch_msgs_tensors", [(a, t, T.ROWS, 32) for a, t in (("R", R), ("S", S), ("A", A))] +
                         [("msgs", msgs, T.BYTES, 0), ("msg_off", msg_off, T.OFF, 0)])
        st = T.empty(dev, n)
        T.launch("eb200_eddsa_verify_batch_msgs_dev", dev, [n, R, S, A, msgs, msgs.numel(), msg_off, st],
                 T.ws_unkeyed(nat.CURVE_ED25519, n))
        return st

    def sign_batch_tensors(self, secrets, msgs, msg_off, want_pub=False):
        """sign_batch_packed on CUDA tensors (eb200_eddsa_sign_batch_dev): secrets (n, 32), the messages back to back in
        msgs (1-D uint8) with (n + 1,) int64 offsets.  Returns (sig (n, 64), status), or (sig, pub (n, 32), status) with
        want_pub; a range that decreases or ends past msgs gets ST_BAD_ITEM and zeroed rows."""
        from . import _tensors as T
        n, dev = T.check("sign_batch_tensors", [("secrets", secrets, T.ROWS, 32), ("msgs", msgs, T.BYTES, 0),
                                                ("msg_off", msg_off, T.OFF, 0)])
        sig, pub, st = T.empty(dev, n, 64), T.empty(dev, n, 32) if want_pub else None, T.empty(dev, n)
        T.launch("eb200_eddsa_sign_batch_dev", dev, [n, secrets, msgs, msgs.numel(), msg_off, sig, pub, st],
                 T.ws_unkeyed(nat.CURVE_ED25519, n))
        return (sig, pub, st) if want_pub else (sig, st)


class EDDSA(_EdKeyObjects, _EdTensorForms):
    def __init__(self, curve="ed25519", device=0):
        if curve != "ed25519":
            raise EllipticError("only tested with ed25519 so far")      # eddsa/index.js:12
        self.encoding_length = 32
        self.n = N_ED25519
        self._device = device

    def hash_int(self, *parts):
        """EDDSA.hashInt (eddsa/index.js:65-70)."""
        h = hashlib.sha512()
        for p in parts:
            h.update(bytes(p))
        return int.from_bytes(h.digest(), "little") % self.n

    def verify_batch_packed(self, R, S, A, h):
        """R, S, A, h: (n, 32) uint8 arrays (little-endian wire forms; h = hashInt(R, A, M) < n)."""
        lib = nat.init(self._device)
        R, S, A, h = (np.ascontiguousarray(a, dtype=np.uint8) for a in (R, S, A, h))
        n = R.shape[0]
        if not (R.shape == (n, 32) and S.shape == R.shape and A.shape == R.shape and h.shape == R.shape):
            raise ValueError("R, S, A, h must be (n, 32) uint8 arrays")
        status = np.empty(n, np.uint8)
        nat.call(lib.eb200_eddsa_verify_batch, n, R, S, A, h, status)
        return status

    def verify_batch_msgs_packed(self, R, S, A, msgs, msg_off):
        """Like verify_batch_packed but takes the raw messages (concatenated bytes + n+1 offsets);
        SHA-512 and the reduction mod n run on the GPU."""
        lib = nat.init(self._device)
        R, S, A = (np.ascontiguousarray(a, dtype=np.uint8) for a in (R, S, A))
        msgs = np.ascontiguousarray(msgs, dtype=np.uint8)
        msg_off = np.ascontiguousarray(msg_off, dtype=np.uint64)
        n = R.shape[0]
        if not (R.shape == (n, 32) and S.shape == R.shape and A.shape == R.shape):
            raise ValueError("R, S, A must be (n, 32) uint8 arrays")
        if not (msg_off.shape == (n + 1,) and int(msg_off[n]) == msgs.size):
            raise ValueError("msg_off must hold n + 1 offsets, the last one equal to len(msgs)")
        status = np.empty(n, np.uint8)
        nat.call(lib.eb200_eddsa_verify_batch_msgs, n, R, S, A, msgs if msgs.size else None, msg_off, status)
        return status

    def _signature(self, sig):
        sig = _parse_bytes(sig)
        if len(sig) != 2 * self.encoding_length:
            raise EllipticError("Signature has invalid size")       # eddsa/signature.js:23-24
        return sig

    def _pub(self, pub):
        pub = _parse_bytes(pub)
        if len(pub) != self.encoding_length:
            # decodePoint on another length reads a different y; not on the accelerated path
            raise EllipticError("unsupported public key length %d" % len(pub))
        return pub

    def verify_batch(self, messages, sigs, pubs, gpu_hash=True):
        """EDDSA#verifyBatch: lists of the reference's own argument forms (hex strings / byte arrays).
        gpu_hash=False computes hashInt with hashlib on the host instead of on the GPU."""
        n = len(messages)
        rsa, ms = [], []
        for i in range(n):
            if not gpu_hash:
                ms.append(_parse_bytes(messages[i]))      # the host path reads the message first
            sig = self._signature(sigs[i])
            pub = self._pub(pubs[i])
            rsa.append(sig + pub)
            if gpu_hash:
                ms.append(_parse_bytes(messages[i]))
        rows = _blob(rsa)[0].reshape(n, 96)
        R, S, A = rows[:, :32], rows[:, 32:64], rows[:, 64:]
        if gpu_hash:
            return self.verify_batch_msgs_packed(R, S, A, *_blob(ms))
        return self.verify_batch_packed(R, S, A, _pack([self.hash_int(x[:32], x[64:], m) for x, m in zip(rsa, ms)], 32, "little"))

    def sign_batch_packed(self, secrets, msgs, msg_off, want_pub=False):
        """secrets: (n, 32) uint8; msgs: concatenated message bytes; msg_off: n + 1 uint64 offsets.
        Returns the (n, 64) signatures Rencoded || S (and the (n, 32) public keys with want_pub)."""
        lib = nat.init(self._device)
        secrets = np.ascontiguousarray(secrets, dtype=np.uint8)
        msgs = np.ascontiguousarray(msgs, dtype=np.uint8)
        msg_off = np.ascontiguousarray(msg_off, dtype=np.uint64)
        n = secrets.shape[0]
        if secrets.shape != (n, 32) or msg_off.shape != (n + 1,) or int(msg_off[n]) != msgs.size:
            raise EllipticError("sign_batch_packed: secrets (n, 32), n + 1 offsets covering msgs expected")
        sig = np.empty((n, 64), np.uint8)
        pub = np.empty((n, 32), np.uint8) if want_pub else None
        st = np.empty(n, np.uint8)
        nat.call(lib.eb200_eddsa_sign_batch, n, secrets, msgs if msgs.size else None, msg_off, sig, pub, st)
        if not bool((st == nat.ST_TRUE).all()):
            raise nat.NativeError("eddsa sign: unexpected status")
        return (sig, pub) if want_pub else sig

    def sign_batch(self, messages, secrets):
        """EDDSA#signBatch: lists of the reference's own argument forms (hex strings / byte arrays); secrets as
        eddsa.keyFromSecret takes them.  Returns a list of 64-byte signatures (sig.toBytes())."""
        n = len(messages)
        sks, ms = [], []
        for i in range(n):
            sk = _parse_bytes(secrets[i])
            if len(sk) != 32:
                raise EllipticError("unsupported secret length %d" % len(sk))
            sks.append(sk)
            ms.append(_parse_bytes(messages[i]))
        sig = self.sign_batch_packed(_blob(sks)[0].reshape(n, 32), *_blob(ms))
        return [sig[i].tobytes() for i in range(n)]

    def sign(self, message, secret):
        """EDDSA.prototype.sign (eddsa/index.js:34-44): the 64 signature bytes (sig.toBytes())."""
        return self.sign_batch([message], [secret])[0]

    def public_from_secret_batch(self, secrets):
        """key.getPublic('bytes') for a batch of secrets (a fixed-base multiplication each)."""
        secrets = np.ascontiguousarray(secrets, dtype=np.uint8)
        n = secrets.shape[0]
        _, pub = self.sign_batch_packed(secrets, np.zeros(0, np.uint8), np.zeros(n + 1, np.uint64), want_pub=True)
        return pub

    def verify(self, message, sig, pub):
        """EDDSA.prototype.verify (eddsa/index.js:52-63): bool, or raises."""
        st = int(self.verify_batch([message], [sig], [pub])[0])
        return _answer(st == nat.ST_TRUE, st, (nat.ST_TRUE, nat.ST_FALSE))


class EdKeySet(_NativeSets):
    """ed25519 public keys imported once and kept on the GPU, raw bytes and per-key tables (eb200_eddsa_keyset_create);
    item i of a verify call is checked against key key_idx[i], with the status EDDSA.verify_batch gives for that key.
    `status`: per key, ST_TRUE (the key decodes) or the throw of decoding it.  close() frees the device memory; the
    object is a context manager."""

    def __init__(self, ed, pubs, table_bits=0):
        self._ed = ed
        A = np.frombuffer(b"".join(ed._pub(p) for p in pubs), np.uint8).reshape(len(pubs), 32).copy()
        self._A = A
        lib = nat.init(ed._device)
        m = len(pubs)
        self.status = np.zeros(m, np.uint8)
        h = ctypes.c_void_p()
        nat.check(lib.eb200_eddsa_keyset_create(m, A.ctypes.data, table_bits, self.status.ctypes.data, ctypes.byref(h)))
        self._sets = [h]
        w, db = ctypes.c_uint32(), ctypes.c_size_t()
        nat.check(lib.eb200_keyset_info(h, None, None, ctypes.byref(w), ctypes.byref(db)))
        self.table_bits, self.device_bytes = w.value, db.value

    def _args(self, R, S, key_idx):
        R, S = (np.ascontiguousarray(a, dtype=np.uint8) for a in (R, S))
        key_idx = np.asarray(key_idx)
        n = R.shape[0]
        if not (R.shape == (n, 32) and S.shape == R.shape and key_idx.shape == (n,)):
            raise ValueError("R, S must be (n, 32) uint8 arrays and key_idx (n,)")
        if n and (key_idx.min() < 0 or key_idx.max() >= len(self.status)):
            raise ValueError("key_idx out of range")
        return R, S, np.ascontiguousarray(key_idx, np.uint32), n

    def _handle(self):
        if not self._sets:
            raise EllipticError("key set is closed")
        return self._sets[0]

    def verify_batch_packed(self, R, S, h, key_idx):
        """R, S, h: (n, 32) uint8 arrays (little-endian wire forms; h = hashInt(R, A, M) < n); key_idx: n indices into
        the set.  Returns the status bytes."""
        R, S, key_idx, n = self._args(R, S, key_idx)
        h = np.ascontiguousarray(h, dtype=np.uint8)
        if h.shape != (n, 32):
            raise ValueError("h must be an (n, 32) uint8 array")
        status = np.empty(n, np.uint8)
        if n:
            nat.call(nat.load().eb200_eddsa_verify_batch_keyed, self._handle(), n, R, S, h, key_idx, status)
        return status

    def verify_batch_msgs_packed(self, R, S, msgs, msg_off, key_idx):
        """Like verify_batch_packed but takes the raw messages (concatenated bytes + n+1 offsets); the key bytes are
        gathered, hashed with R and the message, and reduced mod n on the GPU."""
        R, S, key_idx, n = self._args(R, S, key_idx)
        msgs = np.ascontiguousarray(msgs, dtype=np.uint8)
        msg_off = np.ascontiguousarray(msg_off, dtype=np.uint64)
        if not (msg_off.shape == (n + 1,) and int(msg_off[n]) == msgs.size):
            raise ValueError("msg_off must hold n + 1 offsets, the last one equal to len(msgs)")
        status = np.empty(n, np.uint8)
        if n:
            nat.call(nat.load().eb200_eddsa_verify_batch_keyed_msgs, self._handle(), n, R, S, msgs if msgs.size else None,
                     msg_off, key_idx, status)
        return status

    def verify_batch(self, messages, sigs, key_idx, gpu_hash=True):
        """Lists of the reference's message and signature forms, as EDDSA.verify_batch takes them, against keys of the
        set.  gpu_hash=False computes hashInt with hashlib on the host (over the key's raw bytes) instead."""
        ed, n = self._ed, len(messages)
        if len(sigs) != n or len(key_idx) != n:
            raise ValueError("messages, sigs and key_idx must have the same length")
        ms, sig = [], []
        for i in range(n):                                # each item read in EDDSA.verify_batch's order
            if not gpu_hash:
                ms.append(_parse_bytes(messages[i]))
            sig.append(ed._signature(sigs[i]))
            if gpu_hash:
                ms.append(_parse_bytes(messages[i]))
        rs = np.frombuffer(b"".join(sig), np.uint8).reshape(n, 64)
        if gpu_hash:
            return self.verify_batch_msgs_packed(rs[:, :32], rs[:, 32:], *_blob(ms), key_idx)
        R, S, idx, _ = self._args(rs[:, :32], rs[:, 32:], key_idx)
        h = _pack([ed.hash_int(sig[i][:32], self._A[idx[i]], ms[i]) for i in range(n)], 32, "little")
        return self.verify_batch_packed(R, S, h, idx)

    # ---- tensor forms: the keyed device-buffer calls on CUDA tensors (conventions: _tensors) -------------------------
    def _keyed_tensors(self, name, fn, specs, ins, key_idx, outs):
        from . import _tensors as T
        n, dev = T.check(name, specs + [("key_idx", key_idx, T.IDX, 0)], self._sets)
        return T.keyed(name, self._sets, len(self.status), None, fn, n, dev, ins, key_idx, [(n,) + o for o in outs])

    def verify_batch_tensors(self, R, S, h, key_idx):
        """verify_batch_packed on CUDA tensors (eb200_eddsa_verify_batch_keyed_dev): R, S, h (n, 32); an h >= n gets
        ST_BAD_ITEM.  Returns the statuses."""
        from . import _tensors as T
        (st,) = self._keyed_tensors("verify_batch_tensors", "eb200_eddsa_verify_batch_keyed_dev",
                                    [(a, t, T.ROWS, 32) for a, t in (("R", R), ("S", S), ("h", h))], [R, S, h], key_idx, [])
        return st

    def verify_batch_msgs_tensors(self, R, S, msgs, msg_off, key_idx):
        """verify_batch_msgs_packed on CUDA tensors (eb200_eddsa_verify_batch_keyed_msgs_dev): R, S (n, 32), the messages
        back to back in msgs (1-D uint8) with (n + 1,) int64 offsets.  Returns the statuses."""
        from . import _tensors as T
        specs = [("R", R, T.ROWS, 32), ("S", S, T.ROWS, 32), ("msgs", msgs, T.BYTES, 0), ("msg_off", msg_off, T.OFF, 0)]
        (st,) = self._keyed_tensors("verify_batch_msgs_tensors", "eb200_eddsa_verify_batch_keyed_msgs_dev", specs,
                                    [R, S, msgs, msgs.numel(), msg_off], key_idx, [])
        return st


class EdSigningSet(_NativeSets):
    """ed25519 signing keys imported once from their 32-byte secrets (eb200_eddsa_signing_set_create): the GPU keeps each
    key's clamped scalar, message prefix and encoded public key, and item i of a sign call is signed by key key_idx[i],
    with the bytes EDDSA.sign_batch gives for that key's secret.  The object does not keep the secrets.  `public`: the
    (m, 32) encoded public keys (key.getPublic('bytes')).  close() frees the device memory; the object is a context
    manager."""

    def __init__(self, ed, secrets):
        self._ed = ed
        sks = []
        for s in secrets:
            sk = _parse_bytes(s)
            if len(sk) != 32:
                raise EllipticError("unsupported secret length %d" % len(sk))
            sks.append(sk)
        m = len(sks)
        sec = np.frombuffer(b"".join(sks), np.uint8).reshape(m, 32).copy()
        lib = nat.init(ed._device)
        self.public = np.zeros((m, 32), np.uint8)
        h = ctypes.c_void_p()
        try:
            nat.check(lib.eb200_eddsa_signing_set_create(m, sec.ctypes.data, self.public.ctypes.data, ctypes.byref(h)))
        finally:
            sec[:] = 0
        self._sets = [h]
        db = ctypes.c_size_t()
        nat.check(lib.eb200_keyset_info(h, None, None, None, ctypes.byref(db)))
        self.device_bytes = db.value

    def _handle(self):
        if not self._sets:
            raise EllipticError("signing set is closed")
        return self._sets[0]

    def sign_batch_packed(self, msgs, msg_off, key_idx):
        """msgs: concatenated message bytes; msg_off: n + 1 uint64 offsets; key_idx: n indices into the set.
        Returns the (n, 64) signatures Rencoded || S."""
        msgs = np.ascontiguousarray(msgs, dtype=np.uint8)
        msg_off = np.ascontiguousarray(msg_off, dtype=np.uint64)
        key_idx = np.asarray(key_idx)
        n = key_idx.shape[0] if key_idx.ndim == 1 else -1
        if n < 0 or not (msg_off.shape == (n + 1,) and int(msg_off[n]) == msgs.size):
            raise ValueError("key_idx must be (n,) and msg_off hold n + 1 offsets, the last one equal to len(msgs)")
        if n and (key_idx.min() < 0 or key_idx.max() >= len(self.public)):
            raise ValueError("key_idx out of range")
        sig = np.empty((n, 64), np.uint8)
        if n:
            h, st = self._handle(), np.empty(n, np.uint8)
            nat.call(nat.load().eb200_eddsa_sign_batch_keyed, h, n, msgs if msgs.size else None, msg_off,
                     np.ascontiguousarray(key_idx, np.uint32), sig, st)
            if not bool((st == nat.ST_TRUE).all()):
                raise nat.NativeError("eddsa sign: unexpected status")
        return sig

    def sign_batch(self, messages, key_idx):
        """Messages in the reference's forms (hex strings / byte arrays), as EDDSA.sign_batch takes them, each signed by
        key key_idx[i] of the set.  Returns a list of 64-byte signatures (sig.toBytes())."""
        n = len(messages)
        if len(key_idx) != n:
            raise ValueError("messages and key_idx must have the same length")
        sig = self.sign_batch_packed(*_blob([_parse_bytes(m) for m in messages]), key_idx)
        return [sig[i].tobytes() for i in range(n)]

    def sign_batch_tensors(self, msgs, msg_off, key_idx):
        """sign_batch_packed on CUDA tensors (eb200_eddsa_sign_batch_keyed_dev): the messages back to back in msgs (1-D
        uint8) with (n + 1,) int64 offsets, key_idx (n,).  Returns (sig (n, 64), status)."""
        from . import _tensors as T
        n, dev = T.check("sign_batch_tensors", [("key_idx", key_idx, T.IDX, 0), ("msgs", msgs, T.BYTES, 0),
                                                ("msg_off", msg_off, T.OFF, 0)], self._sets)
        return T.keyed("sign_batch_tensors", self._sets, len(self.public), None, "eb200_eddsa_sign_batch_keyed_dev",
                       n, dev, [msgs, msgs.numel(), msg_off], key_idx, [(n, 64)])
