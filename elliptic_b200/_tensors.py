"""Tensor forms of the device-buffer calls: the `*_tensors` methods of EC, EDDSA, KeySet, EdKeySet, EdSigningSet and
X25519KeySet take PyTorch CUDA tensors, run the C ABI's `eb200_*_dev` call on the caller's stream and return CUDA
tensors, so a pipeline whose data is already on the GPU never copies it to the host.

Conventions, checked before any launch (a violation raises ValueError, a closed key set EllipticError, and nothing is
launched):

- Data.  A fixed-width field is a torch.uint8 tensor of shape (n, len) in the C call's byte order (big-endian ECDSA
  scalars and coordinates, little-endian EdDSA wire forms).  Messages and DER signatures are one 1-D uint8 tensor with
  (n + 1,) int64 offsets into it, passed to the C call as its uint64 offsets; a bad range is the C call's BAD_ITEM.
- Key indices.  key_idx is int32 or int64 of shape (n,).  An index that is negative or not below the set's size gets
  ST_BAD_KEY_INDEX and zeroed outputs: an int64 index is clamped to [-1, m] on the device before it is narrowed to 32
  bits (2^32 + 3 becomes m, not key 3; -1 reads as 2^32 - 1), and a negative int32 index reads as at least 2^31 in the
  C call's uint32.  No
  index is used to address a tensor before it is clamped.
- Device.  Every tensor is contiguous and on one CUDA device, on which the library is then initialised.
- Stream.  The call runs on torch.cuda.current_stream(device); choose another with `with torch.cuda.stream(s):`.
- Workspace.  torch.empty from the caching allocator on that stream, sized by eb200_dev_workspace_bytes or
  eb200_keyset_dev_workspace_bytes, and dropped once the call is enqueued: the allocator only hands the block to later
  work on the same stream.
- Outputs.  New tensors on the device, with the (n,) uint8 status last, returned without a synchronisation.  A sign
  with explicit nonces leaves the r, s and recid of a RETRY item unwritten, so those outputs start zeroed.
- torch is imported here, and this module only by the tensor methods: `import elliptic_b200` does not import torch.

A KeySet that holds one native set per wire format runs one pass per native set, all on the stream: the items of the
other native sets get an index the pass screens out, and each pass's rows are merged into the result where they belong.
"""
import ctypes

from . import _native as nat
from .ec import EllipticError

ROWS, VEC, IDX, BYTES, OFF = "rows", "vec", "idx", "bytes", "off"


def _torch():
    import torch
    return torch


def check(name, specs, sets=None):
    """Checks (arg, tensor, kind, width) specs in order, then their devices, and returns (n, device).  kind: ROWS =
    uint8 (n, width) (width None: any width >= 1), VEC = uint8 (n,), IDX = int32 / int64 (n,), BYTES = uint8 1-D, OFF =
    int64 (n + 1,).  n is the leading size of the first ROWS / VEC / IDX tensor; a tensor given as None is skipped.  sets: a key set's native
    handles, which must not be closed."""
    if sets is not None and not sets:
        raise EllipticError("%s: key set is closed" % name)
    torch = _torch()
    n = None
    dev = None
    for arg, t, kind, width in specs:
        if t is None:
            continue
        if not isinstance(t, torch.Tensor):
            raise ValueError("%s: %s must be a torch.Tensor" % (name, arg))
        want = (torch.int32, torch.int64) if kind == IDX else (torch.int64,) if kind == OFF else (torch.uint8,)
        if t.dtype not in want:
            raise ValueError("%s: %s must be %s, got %s" % (name, arg, " or ".join(map(str, want)), t.dtype))
        if n is None and kind in (ROWS, VEC, IDX) and t.dim() >= 1:
            n = t.shape[0]
        ok = {ROWS: t.dim() == 2 and t.shape[0] == n and (t.shape[1] == width if width else t.shape[1] >= 1),
              VEC: t.dim() == 1 and t.shape[0] == n, IDX: t.dim() == 1 and t.shape[0] == n, BYTES: t.dim() == 1,
              OFF: t.dim() == 1 and n is not None and t.shape[0] == n + 1}[kind]
        if not ok:
            shape = {ROWS: "(n, %s)" % (width or "k"), VEC: "(n,)", IDX: "(n,)", BYTES: "1-D", OFF: "(n + 1,)"}[kind]
            raise ValueError("%s: %s must be %s with n = %s, got %s" % (name, arg, shape, n, tuple(t.shape)))
        if not t.is_contiguous():
            raise ValueError("%s: %s must be contiguous" % (name, arg))
    for arg, t, _, _ in specs:
        if t is None:
            continue
        if t.device.type != "cuda":
            raise ValueError("%s: %s must be on a CUDA device, got %s" % (name, arg, t.device))
        if dev is None:
            dev = t.device
        elif t.device != dev:
            raise ValueError("%s: every tensor must be on one device (%s and %s)" % (name, dev, t.device))
    return n, dev


def empty(dev, *shape):
    return _torch().empty(shape, dtype=_torch().uint8, device=dev)


def zeros(dev, *shape):
    return _torch().zeros(shape, dtype=_torch().uint8, device=dev)


def _arg(a):
    if a is None or isinstance(a, (int, ctypes.c_void_p)):         # NULL, a size, a key set's handle
        return a
    return ctypes.c_void_p(a.data_ptr())


def launch(fn, dev, args, ws_bytes=None):
    """The C call named fn, fn(*args[, workspace], stream), on the current stream of `dev`: tensors pass as their device
    addresses, None as NULL, ints and key-set handles as they are.  ws_bytes: the workspace's size, allocated on that stream, or None when the call takes no
    workspace or args ends with one."""
    torch = _torch()
    lib = nat.init(dev.index)
    fn = getattr(lib, fn)
    stream = torch.cuda.current_stream(dev)
    tail = []
    if ws_bytes is not None:
        tail.append(_arg(empty(dev, ws_bytes)) if ws_bytes else None)
    nat.check(fn(*(_arg(a) for a in args), *tail, ctypes.c_void_p(stream.cuda_stream)))


def ws_unkeyed(curve, n):
    return nat.load().eb200_dev_workspace_bytes(curve, n)


def ws_keyed(h, n):
    return nat.load().eb200_keyset_dev_workspace_bytes(h, n)


def narrow_index(key_idx, m):
    """key_idx as the C call's uint32 indices for a set of m < 2^32 keys, every invalid one >= m: int32 as it is (a
    negative index reads as >= 2^31 >= m), int64 clamped to [-1, m] on the device before it is narrowed, so an index >= m
    becomes m and a negative one -1, which reads as 2^32 - 1 >= m.  One kernel and the narrowing copy."""
    torch = _torch()
    if key_idx.dtype == torch.int32 and m <= 1 << 31:
        return key_idx
    return key_idx.long().clamp(-1, m).to(torch.int32)


def keyed(name, sets, m, where, fn, n, dev, ins, key_idx, outs):
    """The C call named fn, fn(set, n, *ins, idx, *outs, status, workspace, stream), for key indices into a key set:
    sets are its native handles (check() has refused a closed set), m its size, `where` None for one native set, else a
    callable giving the device tensors (set_of, local, sizes) that map a key to its native set and its index there.  outs: the shapes of the
    output rows, (n, w) each.  Returns the outputs and the status."""
    torch = _torch()
    if len(sets) == 1:
        res = [empty(dev, *shape) for shape in outs] + [empty(dev, n)]
        launch(fn, dev, [sets[0], n, *ins, narrow_index(key_idx, m), *res], ws_keyed(sets[0], n))
        return res
    set_of, local, sizes = where(dev)
    idx = key_idx.long()
    valid = (idx >= 0) & (idx < m)
    safe = torch.where(valid, idx, 0)                  # clamped before it addresses the map
    owner = torch.where(valid, set_of[safe], -1)
    loc = local[safe]
    res = [zeros(dev, *shape) for shape in outs] + [torch.full((n,), nat.ST_BAD_KEY_INDEX, dtype=torch.uint8, device=dev)]
    ws = empty(dev, max(ws_keyed(h, n) for h in sets))     # one workspace for every pass, in stream order
    for s, h in enumerate(sets):
        sel = owner == s
        part = [empty(dev, *shape) for shape in outs] + [empty(dev, n)]
        launch(fn, dev, [h, n, *ins, torch.where(sel, loc, sizes[s]).to(torch.int32), *part, ws])
        res = [torch.where(sel.view(-1, *[1] * (r.dim() - 1)), p, r) for r, p in zip(res, part)]
    return res
