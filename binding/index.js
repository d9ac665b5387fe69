'use strict';
// Drop-in for require('elliptic'): every export of lib/elliptic.js:5-13 is the reference's own object
// (single-item behaviour unchanged); the batch entry points below are added on the same prototypes and
// run on the GPU through the N-API addon -> libelliptic_b200.so (include/elliptic_b200.h):
//   EC#verifyBatch / verifyBatchAsync / signBatch / genKeyPairBatch / recoverPubKeyBatch / getKeyRecoveryParamBatch /
//   deriveBatch
//   EDDSA#verifyBatch / signBatch / keySet / signingSet
//   curve.short#mulBatch / mulAddBatch / addBatch / dblBatch / validateBatch   (any parameters, presets take the tuned kernels)
//   curve.edwards#mulBatch / mulAddBatch (ed25519), curve.mont#mulBatch (curve25519)
// All parsing (hex / byte arrays / DER / SEC1, _truncateToN) is done by the reference's own JS, so accept / reject /
// throw behaviour is the reference's by construction; only fixed-width big-endian arrays cross into the addon.
var elliptic = require('elliptic');
var native = require('./elliptic_b200.node');
var BN = require('bn.js');

var CURVE = { secp256k1: 1, p256: 2, p384: 3, ed25519: 4, curve25519: 5, p521: 6, p192: 7, p224: 8 };
var THROW = { 2: 'invalid point', 3: 'public point not validated', 5: 'Assertion failed', 6: 'Unknown point format',
  8: 'Unable to find sencond key candinate', 9: 'Signature without r or s' };
var inited = false;
// init(devices): CUDA ordinals to use (default: every visible device); batches are sharded over them inside the library
function init(devices) { if (!inited || devices) { native.init(devices, 0); inited = true; } }
elliptic.b200 = { init: init, native: native };

function be(bn, len) { return bn.toArray('be', len); }
function presetName(curve) {
  var names = Object.keys(CURVE);
  for (var i = 0; i < names.length; i++) if (elliptic.curves[names[i]].curve === curve) return names[i];
  return undefined;
}
function curveId(ec) { var n = presetName(ec.curve); return n === undefined ? undefined : CURVE[n]; }
function pack(list, len, f) {
  var out = new Uint8Array(list.length * len);
  list.forEach(function(v, i) { out.set(f(v, i), i * len); });
  return out;
}
function statusToBool(v) { if (v > 1) throw new Error(THROW[v] || ('status ' + v)); return v === 1; }

// ---- EC ------------------------------------------------------------------------------------------------------
function packVerify(ec, msgs, sigs, keys, enc, options) {
  var len = ec.curve.p.byteLength(), n = msgs.length;
  var e = new Uint8Array(n * len), r = new Uint8Array(n * len), s = new Uint8Array(n * len);
  var pub = new Uint8Array(n * 2 * len), early = {};
  var Signature = ec.sign('00', '01').constructor;                   // lib/elliptic/ec/signature.js
  for (var i = 0; i < n; i++) {
    var msg = ec._truncateToN(msgs[i], false, options && options.msgBitLength);     // ec/index.js:192
    var key = ec.keyFromPublic(keys[i], enc).getPublic();             // ec/index.js:193 (may throw, as verify)
    var sig = new Signature(sigs[i], 'hex');                          // ec/index.js:194
    if (sig.r.cmpn(1) < 0 || sig.r.cmp(ec.n) >= 0 || sig.s.cmpn(1) < 0 || sig.s.cmp(ec.n) >= 0) { early[i] = false; continue; }
    e.set(be(msg, len), i * len); r.set(be(sig.r, len), i * len); s.set(be(sig.s, len), i * len);
    pub.set(be(key.getX(), len), 2 * i * len); pub.set(be(key.getY(), len), (2 * i + 1) * len);
  }
  return { e: e, r: r, s: s, pub: pub, early: early };
}
function verdicts(ec, st, p, msgs, sigs, keys, enc, options) {
  var out = new Array(msgs.length);
  for (var i = 0; i < msgs.length; i++) {
    if (i in p.early) out[i] = false;
    else if (st[i] === 4) out[i] = ec.verify(msgs[i], sigs[i], keys[i], enc, options);   // un-validated off-curve Edwards key: reference path
    else out[i] = statusToBool(st[i]);
  }
  return out;
}
// EC#verifyBatch(msgs, sigs, keys[, enc][, options]) -> Array<boolean>; throws where a loop over verify() would.
elliptic.ec.prototype.verifyBatch = function verifyBatch(msgs, sigs, keys, enc, options) {
  var id = curveId(this);
  if (id === undefined || this.curve.type === 'mont')
    return msgs.map(function(m, i) { return this.verify(m, sigs[i], keys[i], enc, options); }, this);
  init();
  var p = packVerify(this, msgs, sigs, keys, enc, options);
  return verdicts(this, native.ecdsaVerifyBatch(id, p.e, p.r, p.s, p.pub, 0), p, msgs, sigs, keys, enc, options);
};
// Promise variant: the GPU call runs on a libuv worker (napi_create_async_work)
elliptic.ec.prototype.verifyBatchAsync = function verifyBatchAsync(msgs, sigs, keys, enc, options) {
  var id = curveId(this), self = this;
  if (id === undefined || this.curve.type === 'mont') return Promise.resolve(this.verifyBatch(msgs, sigs, keys, enc, options));
  init();
  var p = packVerify(this, msgs, sigs, keys, enc, options);
  return native.ecdsaVerifyBatchAsync(id, p.e, p.r, p.s, p.pub, 0).then(function(st) {
    return verdicts(self, st, p, msgs, sigs, keys, enc, options);
  });
};

// EC#verifyBatchWire(hashes, ders, keys) -> Array<boolean>: wire formats straight to the GPU -- `hashes` byte arrays of the
// curve's field length (already what _truncateToN leaves), `ders` DER signatures, `keys` SEC1 keys that all have the
// same form (33-byte compressed or 65-byte / 1 + 2 len uncompressed / hybrid).  Signature._importDER
// (ec/signature.js:73-134) and BaseCurve.decodePoint / pointFromX (base.js:270-292) run on the GPU; an item throws
// exactly where the reference would.
elliptic.ec.prototype.verifyBatchWire = function verifyBatchWire(hashes, ders, keys) {
  var id = curveId(this), self = this, len = this.curve.p.byteLength(), n = hashes.length;
  var klen = n ? keys[0].length : 0, fmt = klen === 1 + len ? 2 : klen === 1 + 2 * len ? 1 : 0;
  if (id === undefined || this.curve.type === 'mont' || !fmt || keys.some(function(k) { return k.length !== klen; }) ||
      hashes.some(function(h) { return h.length !== len; }))
    return hashes.map(function(h, i) { return self.verify(h, ders[i], keys[i]); });
  init();
  var sg = concatMsgs(ders);
  var st = native.ecdsaVerifyBatchDer(id, pack(hashes, len, function(h) { return h; }), sg.blob, sg.off, pack(keys, klen, function(k) { return k; }), fmt);
  return Array.prototype.map.call(st, function(v, i) { return v === 4 ? self.verify(hashes[i], ders[i], keys[i]) : statusToBool(v); });
};

// EC#keySet(pubs[, enc]) -> {status, tableBits, deviceBytes, verifyBatch(msgs, sigs, keyIdx[, options]),
// verifyBatchWire(hashes, ders, keyIdx), mul(keyIdx, ks),
// mulAdd(k1s, keyIdx, k2s), derive(privs, keyIdx), getKeyRecoveryParam(msgs, sigs, keyIdx[, enc]), destroy()}: the batch
// form of `key = ec.keyFromPublic(pub, enc); key.getPublic().precompute()` once and key.verify(msg, sig), pub.mul(k),
// G.mulAdd(k1, pub, k2) (Arrays of Points), keyPair.derive(pub) (an Array of BN) and
// ec.getKeyRecoveryParam(msg, sig, pub) (an Array of numbers, throwing where a loop over that call would) many times.
// verifyBatchWire is the keyed EC#verifyBatchWire: hashes of the field length and DER signatures, parsed on the GPU.
// The keys are imported here (a key that throws, throws here, as keyFromPublic does) and kept on the GPU with their
// tables.  mul and mulAdd take their scalars as Short#mulBatch and Short#mulAddBatch do, and an off-curve key's result
// is theirs for that point, not the reference's precomputed-point schedule.
elliptic.ec.prototype.keySet = function keySet(pubs, enc) {
  var id = curveId(this), self = this, len = this.curve.p.byteLength();
  if (id !== undefined && this.curve.type === 'mont') return x25519KeySet(this, pubs, enc);
  if (id === undefined || this.curve.type !== 'short') throw new Error('key sets: short preset curves only');
  init();
  var keys = pubs.map(function(k) { return self.keyFromPublic(k, enc); });
  var xy = pack(keys, 2 * len, function(k) { var P = k.getPublic(); return be(P.getX(), len).concat(be(P.getY(), len)); });
  var set = native.keysetCreate(id, xy, 0, 0);
  var Signature = this.sign('00', '01').constructor;
  return {
    status: set.status, tableBits: set.tableBits, deviceBytes: set.deviceBytes,
    verifyBatch: function(msgs, sigs, keyIdx, options) {
      var n = msgs.length, e = new Uint8Array(n * len), r = new Uint8Array(n * len), s = new Uint8Array(n * len), early = {};
      var idx = new Uint32Array(n);
      for (var i = 0; i < n; i++) {
        if (!(keyIdx[i] >= 0 && keyIdx[i] < keys.length)) throw new Error('key index out of range');
        idx[i] = keyIdx[i];
        var msg = self._truncateToN(msgs[i], false, options && options.msgBitLength);
        var sig = new Signature(sigs[i], 'hex');
        if (sig.r.cmpn(1) < 0 || sig.r.cmp(self.n) >= 0 || sig.s.cmpn(1) < 0 || sig.s.cmp(self.n) >= 0) { early[i] = false; continue; }
        e.set(be(msg, len), i * len); r.set(be(sig.r, len), i * len); s.set(be(sig.s, len), i * len);
      }
      var st = native.ecdsaVerifyBatchKeyed(set.handle, e, r, s, new Uint8Array(idx.buffer));
      return Array.prototype.map.call(st, function(v, i) { return i in early ? false : statusToBool(v); });
    },
    verifyBatchWire: function(hashes, ders, keyIdx) {
      if (hashes.some(function(h) { return h.length !== len; })) throw new Error('verifyBatchWire: hashes of ' + len + ' bytes');
      var idx = keyIndices(keyIdx), sg = concatMsgs(ders);
      var st = native.ecdsaVerifyBatchKeyedDer(set.handle, pack(hashes, len, function(h) { return h; }), sg.blob, sg.off, idx);
      return Array.prototype.map.call(st, function(v) { return statusToBool(v); });
    },
    mul: function(keyIdx, ks) {
      var big = new BN(1).ushln(8 * len);          // Short#mulBatch's rule: only a k of 2^(8 len) or more is reduced mod n
      var k = pack(ks, len, function(v) { v = new BN(v, 16); return be(v.cmp(big) >= 0 ? v.umod(self.n) : v, len); });
      return pointsOut(self.curve, native.mulAddBatchKeyed(set.handle, null, k, keyIndices(keyIdx)), ks.length, len);
    },
    mulAdd: function(k1s, keyIdx, k2s) {
      return pointsOut(self.curve, native.mulAddBatchKeyed(set.handle, pack(k1s, len, scalar), pack(k2s, len, scalar), keyIndices(keyIdx)),
        k1s.length, len);
    },
    derive: function(privs, keyIdx) {
      var res = native.ecdhDeriveBatchKeyed(set.handle, pack(privs, len, scalar), keyIndices(keyIdx)), out = [];
      for (var i = 0; i < privs.length; i++) {
        if (res.status[i] !== 1) throw new Error(THROW[res.status[i]]);
        out.push(new BN(res.out.subarray(len * i, len * i + len)));
      }
      return out;
    },
    getKeyRecoveryParam: function(msgs, sigs, keyIdx, enc) {
      var n = msgs.length, idx = new Uint32Array(keyIndices(keyIdx).buffer);
      var S = sigs.map(function(s) { return new Signature(s, enc); });
      var one = function(i) { return self.getKeyRecoveryParam(msgs[i], sigs[i], keys[idx[i]].getPublic(), enc); };
      if (S.some(function(s) { return s.r.byteLength() > len; })) return msgs.map(function(_, i) { return one(i); });
      var todo = [];
      S.forEach(function(s, i) { if (s.recoveryParam === null) todo.push(i); });
      var res = null;
      if (todo.length) {
        var e = pack(todo, len, function(i) { return be(new BN(msgs[i]).umod(self.n), len); });
        var r = pack(todo, len, function(i) { return be(S[i].r, len); });
        var s = pack(todo, len, function(i) { return be(S[i].s.umod(self.n), len); });
        var ti = Uint32Array.from(todo, function(i) { return idx[i]; });
        res = native.ecdsaRecoveryParamBatchKeyed(set.handle, e, r, s, new Uint8Array(ti.buffer));
      }
      var out = new Array(n), k = 0;
      for (var i = 0; i < n; i++) {
        if (k < todo.length && todo[k] === i) {
          if (res.status[k] !== 1) throw new Error('Unable to find valid recovery factor');
          out[i] = res.recid[k++];
        } else out[i] = one(i);
      }
      return out;
    },
    destroy: function() { native.keysetDestroy(set.handle); }
  };
  function scalar(v) { return be(new BN(v, 16).umod(self.n), len); }
  function keyIndices(keyIdx) {
    var idx = new Uint32Array(keyIdx.length);
    for (var i = 0; i < keyIdx.length; i++) {
      if (!(keyIdx[i] >= 0 && keyIdx[i] < keys.length)) throw new Error('key index out of range');
      idx[i] = keyIdx[i];
    }
    return new Uint8Array(idx.buffer);
  }
};

// EC#keySet(pubs[, enc]) on curve25519 -> {status, tableBits, deviceBytes, derive(privs, keyIdx), destroy()}: the batch
// form of `pub = ec.keyFromPublic(x, enc)` once and keyPair.derive(pub) (an Array of BN, throwing where a loop over derive
// would) many times.  A key on the twist imports, as keyFromPublic does (status 5), and its derives throw
// 'Assertion failed'.  The GPU keeps each key as its edwards25519 image with a per-key table.
function x25519KeySet(ec, pubs, enc) {
  init();
  var keys = pubs.map(function(k) { return ec.keyFromPublic(k, enc); });
  var set = native.x25519KeysetCreate(pack(keys, 32, function(k) { return be(k.getPublic().getX(), 32); }), 0);
  return {
    status: set.status, tableBits: set.tableBits, deviceBytes: set.deviceBytes,
    derive: function(privs, keyIdx) {
      if (privs.length !== keyIdx.length) throw new Error('one key index per private key');
      var idx = new Uint32Array(privs.length), out = [];
      for (var i = 0; i < privs.length; i++) {
        if (!(keyIdx[i] >= 0 && keyIdx[i] < keys.length)) throw new Error('key index out of range');
        idx[i] = keyIdx[i];
      }
      var k = pack(privs, 32, function(p) { return be(ec.keyFromPrivate(p).getPrivate(), 32); });
      var res = native.x25519DeriveBatchKeyed(set.handle, k, new Uint8Array(idx.buffer));
      for (i = 0; i < privs.length; i++) {
        if (res.status[i] !== 1) throw new Error(THROW[res.status[i]]);
        out.push(new BN(res.out.subarray(32 * i, 32 * i + 32)));
      }
      return out;
    },
    destroy: function() { native.keysetDestroy(set.handle); }
  };
}

// EC#signBatch(msgs, keys[, enc][, options]) -> Array<Signature>.  options: canonical, pers / persEnc (one string for the
// batch), k: function(item, iter) -> BN (the reference's options.k per item), msgBitLength.
elliptic.ec.prototype.signBatch = function signBatch(msgs, keys, enc, options) {
  if (typeof enc === 'object') { options = enc; enc = null; }
  options = options || {};
  var id = curveId(this), self = this;
  if (id === undefined || this.curve.type === 'mont')
    return msgs.map(function(m, i) { return this.sign(m, keys[i], enc, options); }, this);
  init();
  var len = this.n.byteLength(), n = msgs.length, Signature = this.sign('00', '01').constructor;
  var e = pack(msgs, len, function(m) { return be(self._truncateToN(m, false, options.msgBitLength), len); });   // ec/index.js:126
  var d = pack(keys, len, function(k) { return be(self.keyFromPrivate(k, enc).getPrivate(), len); });
  var flags = options.canonical ? 1 : 0, out = new Array(n);
  function take(res, idx) {
    var again = [];
    idx.forEach(function(i, j) {
      if (res.status[j] === 10) { again.push(i); return; }           // the reference's loop `continue`s: next k(iter)
      if (res.status[j] !== 1) throw new Error('sign status ' + res.status[j]);
      out[i] = new Signature({ r: new BN(res.r.subarray(len * j, len * j + len)), s: new BN(res.s.subarray(len * j, len * j + len)),
        recoveryParam: res.recid[j] });
    });
    return again;
  }
  var all = msgs.map(function(_, i) { return i; });
  if (options.k) {
    var todo = all;
    for (var iter = 0; todo.length; iter++) {
      var k = pack(todo, len, function(i) {
        var kv = self._truncateToN(options.k(i, iter), true);        // ec/index.js:154-157
        return be(kv, len);
      });
      var sub = function(a) { return pack(todo, len, function(i) { return a.subarray(len * i, len * i + len); }); };
      todo = take(native.ecdsaSignBatch(id, sub(e), sub(d), flags, k, null), todo);
    }
  } else {
    var pers = options.pers === undefined ? null : Uint8Array.from(elliptic.utils.toArray(options.pers, options.persEnc || 'utf8'));
    take(native.ecdsaSignBatch(id, e, d, flags, null, pers), all);
  }
  return out;
};

// EC#genKeyPairBatch(entropies[, options]) -> Array<KeyPair>  (genKeyPair({entropy, entropyEnc, pers, persEnc}), ec/index.js:55-79)
elliptic.ec.prototype.genKeyPairBatch = function genKeyPairBatch(entropies, options) {
  options = options || {};
  var id = curveId(this), self = this;
  var ents = entropies.map(function(x) { return elliptic.utils.toArray(x, options.entropyEnc || 'utf8'); });
  var elen = ents.length ? ents[0].length : 0;
  if (id === undefined || this.curve.type === 'mont' || ents.some(function(x) { return x.length !== elen || x.length < 24; }))
    return entropies.map(function(x) { return self.genKeyPair({ entropy: x, entropyEnc: options.entropyEnc, pers: options.pers, persEnc: options.persEnc }); });
  init();
  var len = this.n.byteLength();
  var pers = options.pers === undefined ? null : Uint8Array.from(elliptic.utils.toArray(options.pers, options.persEnc || 'utf8'));
  var res = native.ecKeygenBatch(id, pack(ents, elen, function(x) { return x; }), elen, pers);
  return ents.map(function(_, i) { return self.keyFromPrivate(new BN(res.priv.subarray(len * i, len * i + len))); });
};

// EC#recoverPubKeyBatch(msgs, sigs, js[, enc]) -> Array<Point>
elliptic.ec.prototype.recoverPubKeyBatch = function recoverPubKeyBatch(msgs, sigs, js, enc) {
  var id = curveId(this), self = this;
  var len = this.curve.p.byteLength(), n = msgs.length;
  var Signature = this.sign('00', '01').constructor;
  var S = sigs.map(function(s) { return new Signature(s, enc); });
  if (id === undefined || this.curve.type !== 'short' || S.some(function(s) { return s.r.byteLength() > len; }))
    return msgs.map(function(m, i) { return self.recoverPubKey(m, sigs[i], js[i], enc); });
  init();
  js.forEach(function(j) { if ((3 & j) !== j) throw new Error('The recovery param is more than two bits'); });
  var e = pack(msgs, len, function(m) { return be(new BN(m).umod(self.n), len); });
  var r = pack(S, len, function(s) { return be(s.r, len); }), s = pack(S, len, function(x) { return be(x.s.umod(self.n), len); });
  var res = native.ecdsaRecoverBatch(id, e, r, s, Uint8Array.from(js));
  var out = [];
  for (var i = 0; i < n; i++) {
    if (res.status[i] === 7) out.push(this.curve.point(null, null));
    else if (res.status[i] !== 1) throw new Error(THROW[res.status[i]]);
    else out.push(this.curve.point(new BN(res.pub.subarray(2 * len * i, 2 * len * i + len)), new BN(res.pub.subarray(2 * len * i + len, 2 * len * (i + 1)))));
  }
  return out;
};

// EC#getKeyRecoveryParamBatch(msgs, sigs, Qs[, enc]) -> Array<number>   (getKeyRecoveryParam, ec/index.js:261-278); throws
// 'Unable to find valid recovery factor' where a loop over getKeyRecoveryParam would.  The reference's own call answers
// wherever recoverPubKeyBatch falls back, and for signatures that carry a recoveryParam or a Q at infinity.
elliptic.ec.prototype.getKeyRecoveryParamBatch = function getKeyRecoveryParamBatch(msgs, sigs, Qs, enc) {
  var id = curveId(this), self = this;
  var len = this.curve.p.byteLength(), n = msgs.length;
  var Signature = this.sign('00', '01').constructor;
  var S = sigs.map(function(s) { return new Signature(s, enc); });
  var one = function(i) { return self.getKeyRecoveryParam(msgs[i], sigs[i], Qs[i], enc); };
  if (id === undefined || this.curve.type !== 'short' || S.some(function(s) { return s.r.byteLength() > len; }))
    return msgs.map(function(_, i) { return one(i); });
  var todo = [];
  S.forEach(function(s, i) { if (s.recoveryParam === null && !Qs[i].isInfinity()) todo.push(i); });
  var res = null;
  if (todo.length) {
    init();
    var e = pack(todo, len, function(i) { return be(new BN(msgs[i]).umod(self.n), len); });
    var r = pack(todo, len, function(i) { return be(S[i].r, len); });
    var s = pack(todo, len, function(i) { return be(S[i].s.umod(self.n), len); });
    var q = pack(todo, 2 * len, function(i) { return be(Qs[i].getX(), len).concat(be(Qs[i].getY(), len)); });
    res = native.ecdsaRecoveryParamBatch(id, e, r, s, q);
  }
  var out = new Array(n), k = 0;
  for (var i = 0; i < n; i++) {
    if (k < todo.length && todo[k] === i) {
      if (res.status[k] !== 1) throw new Error('Unable to find valid recovery factor');
      out[i] = res.recid[k++];
    } else out[i] = one(i);
  }
  return out;
};

// EC#deriveBatch(privs, pubs) -> Array<BN>   (KeyPair.derive, ec/key.js:102-107)
elliptic.ec.prototype.deriveBatch = function deriveBatch(privs, pubs) {
  var id = curveId(this), self = this, n = privs.length, res, i, out = [];
  if (id === undefined) return privs.map(function(p, j) { return self.keyFromPrivate(p).derive(self.keyFromPublic(pubs[j]).getPublic()); });
  init();
  var len = this.curve.p.byteLength();
  var k = pack(privs, len, function(p) { return be(self.keyFromPrivate(p).getPrivate(), len); });
  if (this.curve.type === 'mont') {
    res = native.x25519Batch(k, pack(pubs, len, function(p) { return be(self.keyFromPublic(p).getPublic().getX(), len); }), 1);
  } else {
    res = native.ecdhDeriveBatch(id, k, pack(pubs, 2 * len, function(p) {
      var q = self.keyFromPublic(p).getPublic(); return be(q.getX(), len).concat(be(q.getY(), len));
    }));
  }
  for (i = 0; i < n; i++) {
    if (res.status[i] !== 1) throw new Error(THROW[res.status[i]]);
    out.push(new BN(res.out.subarray(len * i, len * i + len)));
  }
  return out;
};

// ---- EDDSA ---------------------------------------------------------------------------------------------------
function concatMsgs(list) {
  var off = new BigUint64Array(list.length + 1), total = 0;
  list.forEach(function(m, i) { total += m.length; off[i + 1] = BigInt(total); });
  var blob = new Uint8Array(total + 1), at = 0;
  list.forEach(function(m) { blob.set(m, at); at += m.length; });
  return { blob: blob, off: new Uint8Array(off.buffer) };
}
// EDDSA#verifyBatch(messages, sigs, pubs) -> Array<boolean>   (SHA-512 of R || A || M on the GPU)
elliptic.eddsa.prototype.verifyBatch = function verifyBatch(messages, sigs, pubs) {
  init();
  var n = messages.length, R = new Uint8Array(32 * n), S = new Uint8Array(32 * n), A = new Uint8Array(32 * n), ms = [];
  for (var i = 0; i < n; i++) {
    var sig = this.makeSignature(sigs[i]);                             // asserts the size (eddsa/signature.js:23-24)
    var key = this.keyFromPublic(pubs[i]);
    R.set(sig.Rencoded(), 32 * i); S.set(sig.Sencoded(), 32 * i); A.set(key.pubBytes(), 32 * i);
    ms.push(elliptic.utils.parseBytes(messages[i]));
  }
  var m = concatMsgs(ms);
  return Array.prototype.map.call(native.eddsaVerifyBatch(R, S, A, null, m.blob, m.off), statusToBool);
};
// EDDSA#keySet(pubs) -> {status, tableBits, deviceBytes, verifyBatch(messages, sigs, keyIdx), destroy()}: the batch form
// of `key = eddsa.keyFromPublic(pub)` once and eddsa.verify(msg, sig, key) many times.  The keys' bytes (pubBytes(), as
// given for a key made from bytes) are kept on the GPU with their tables; SHA-512 of R || A || M runs there too.
elliptic.eddsa.prototype.keySet = function keySet(pubs) {
  init();
  var self = this;
  var keys = pubs.map(function(k) { return self.keyFromPublic(k); });
  var set = native.eddsaKeysetCreate(pack(keys, 32, function(k) { return k.pubBytes(); }), 0);
  return {
    status: set.status, tableBits: set.tableBits, deviceBytes: set.deviceBytes,
    verifyBatch: function(messages, sigs, keyIdx) {
      var n = messages.length, R = new Uint8Array(32 * n), S = new Uint8Array(32 * n), idx = new Uint32Array(n), ms = [];
      for (var i = 0; i < n; i++) {
        if (!(keyIdx[i] >= 0 && keyIdx[i] < keys.length)) throw new Error('key index out of range');
        idx[i] = keyIdx[i];
        var sig = self.makeSignature(sigs[i]);                         // asserts the size (eddsa/signature.js:23-24)
        R.set(sig.Rencoded(), 32 * i); S.set(sig.Sencoded(), 32 * i);
        ms.push(elliptic.utils.parseBytes(messages[i]));
      }
      var m = concatMsgs(ms);
      return Array.prototype.map.call(native.eddsaVerifyBatchKeyed(set.handle, R, S, null, m.blob, m.off, new Uint8Array(idx.buffer)),
        statusToBool);
    },
    destroy: function() { native.keysetDestroy(set.handle); }
  };
};
// EDDSA#signingSet(secrets) -> {pub, signBatch(messages, keyIdx), destroy()}: the batch form of
// `key = eddsa.keyFromSecret(secret)` once and key.sign(msg) many times.  The GPU keeps each key's clamped scalar, message
// prefix and encoded public key (pub: key.getPublic('bytes') per key), not the secret; signBatch returns Signature objects.
elliptic.eddsa.prototype.signingSet = function signingSet(secrets) {
  var self = this;
  var secs = secrets.map(function(s) { return elliptic.utils.parseBytes(s); });
  if (secs.some(function(s) { return s.length !== 32; })) throw new Error('signing sets take 32-byte secrets');
  init();
  var set = native.eddsaSigningSetCreate(pack(secs, 32, function(s) { return s; }));
  var pubs = [];
  for (var k = 0; k < secs.length; k++) pubs.push(Array.from(set.pub.subarray(32 * k, 32 * k + 32)));
  return {
    pub: pubs,
    signBatch: function(messages, keyIdx) {
      var n = messages.length, idx = new Uint32Array(n);
      for (var i = 0; i < n; i++) {
        if (!(keyIdx[i] >= 0 && keyIdx[i] < pubs.length)) throw new Error('key index out of range');
        idx[i] = keyIdx[i];
      }
      var m = concatMsgs(messages.map(function(x) { return elliptic.utils.parseBytes(x); }));
      var sig = native.eddsaSignBatchKeyed(set.handle, m.blob, m.off, new Uint8Array(idx.buffer));
      return messages.map(function(_, i) { return self.makeSignature(Array.from(sig.subarray(64 * i, 64 * i + 64))); });
    },
    destroy: function() { native.keysetDestroy(set.handle); }
  };
};
// EDDSA#signBatch(messages, secrets) -> Array<Signature>   (eddsa/index.js:34-44; 32-byte secrets)
elliptic.eddsa.prototype.signBatch = function signBatch(messages, secrets) {
  var self = this;
  var secs = secrets.map(function(s) { return elliptic.utils.parseBytes(s); });
  if (secs.some(function(s) { return s.length !== 32; })) return messages.map(function(m, i) { return self.sign(m, secrets[i]); });
  init();
  var m = concatMsgs(messages.map(function(x) { return elliptic.utils.parseBytes(x); }));
  var res = native.eddsaSignBatch(pack(secs, 32, function(s) { return s; }), m.blob, m.off);
  return messages.map(function(_, i) { return self.makeSignature(Array.from(res.sig.subarray(64 * i, 64 * i + 64))); });
};

// ---- .curve ----------------------------------------------------------------------------------------------------
function pointsOut(curve, res, n, len) {
  var out = [];
  for (var i = 0; i < n; i++) {
    if (res.status[i] === 4) throw new Error('point ' + i + ' is not on the curve (the reference does not validate it): use the single-item path');
    out.push(res.status[i] === 1 ? curve.point(new BN(res.points.subarray(2 * len * i, 2 * len * i + len)),
      new BN(res.points.subarray(2 * len * i + len, 2 * len * (i + 1)))) : curve.point(null, null));
  }
  return out;
}
function xy(len) { return function(pt) { return be(pt.getX(), len).concat(be(pt.getY(), len)); }; }
function scalars(ks) {
  var v = ks.map(function(k) { return new BN(k, 16); }), klen = 1;
  v.forEach(function(k) { klen = Math.max(klen, k.byteLength()); });
  return { klen: klen, buf: pack(v, klen, function(k) { return be(k, klen); }) };
}
function rtCall(curve, op, k1, p1, k2, p2) {
  init();
  var len = curve.p.byteLength(), f = xy(len);
  var s = k1 ? scalars(k2 ? k1.concat(k2) : k1) : { klen: 1, buf: null }, n = p1.length;
  var a = be(curve.a.fromRed(), len), b = be(curve.b.fromRed(), len);
  return pointsOut(curve, native.curveOpBatch(op, len, Uint8Array.from(be(curve.p, len)), Uint8Array.from(a), Uint8Array.from(b),
    k1 ? s.buf.subarray(0, n * s.klen) : null, pack(p1, 2 * len, f), k2 ? s.buf.subarray(n * s.klen) : null,
    p2 ? pack(p2, 2 * len, f) : null, s.klen), n, len);
}
var Short = elliptic.curve.short.prototype;
// curve.short#mulBatch(points, scalars) -> Array<Point>   (Point.mul, short.js:422-432; null points: the base point)
Short.mulBatch = function mulBatch(points, ks) {
  var name = presetName(this), len = this.p.byteLength(), n = ks.length, self = this;
  if (name !== undefined) {                                           // tuned preset kernels
    init();
    var big = new BN(1).ushln(8 * len);
    var k = pack(ks, len, function(v) { v = new BN(v, 16); return be(v.cmp(big) >= 0 ? v.umod(self.n) : v, len); });
    return pointsOut(this, native.mulAddBatch(CURVE[name], null, k, points && pack(points, 2 * len, xy(len))), n, len);
  }
  return rtCall(this, 0, ks, points || ks.map(function() { return self.g; }));
};
// curve.short#mulAddBatch(k1s, p2s, k2s) -> Array<Point>   (G.mulAdd(k1, P2, k2), short.js:434-441)
Short.mulAddBatch = function mulAddBatch(k1s, p2s, k2s) {
  var name = presetName(this), len = this.p.byteLength(), self = this;
  if (name !== undefined) {
    init();
    var f = function(v) { return be(new BN(v, 16).umod(self.n), len); };
    return pointsOut(this, native.mulAddBatch(CURVE[name], pack(k1s, len, f), pack(k2s, len, f), pack(p2s, 2 * len, xy(len))), k1s.length, len);
  }
  return rtCall(this, 0, k1s, k1s.map(function() { return self.g; }), k2s, p2s);
};
Short.addBatch = function addBatch(p1s, p2s) { return rtCall(this, 1, null, p1s, null, p2s); };
Short.dblBatch = function dblBatch(ps) { return rtCall(this, 2, null, ps); };
Short.validateBatch = function validateBatch(ps) {
  init();
  var len = this.p.byteLength();
  var res = native.curveOpBatch(3, len, Uint8Array.from(be(this.p, len)), Uint8Array.from(be(this.a.fromRed(), len)),
    Uint8Array.from(be(this.b.fromRed(), len)), null, pack(ps, 2 * len, xy(len)), null, null, 1);
  return Array.prototype.map.call(res.status, function(v) { return v === 1; });
};
// curve.edwards#mulBatch / mulAddBatch on the ed25519 preset (edwards.js:362-375).  The group has order 8n (cofactor 8):
// a point's scalar is reduced mod 8n, which keeps k P for points with a torsion component; G's scalar mod n.
var Edw = elliptic.curve.edwards.prototype;
Edw.mulBatch = function mulBatch(points, ks) {
  var self = this;
  if (presetName(this) !== 'ed25519') return ks.map(function(k, i) { return (points ? points[i] : self.g).mul(new BN(k, 16)); });
  init();
  var n8 = this.n.muln(8);
  var k = pack(ks, 32, function(v) { return be(new BN(v, 16).umod(n8), 32); });
  return pointsOut(this, native.mulAddBatch(CURVE.ed25519, null, k, points && pack(points, 64, xy(32))), ks.length, 32);
};
Edw.mulAddBatch = function mulAddBatch(k1s, p2s, k2s) {
  var self = this;
  if (presetName(this) !== 'ed25519') return k1s.map(function(k, i) { return self.g.mulAdd(new BN(k, 16), p2s[i], new BN(k2s[i], 16)); });
  init();
  var n8 = this.n.muln(8);
  var f = function(v) { return be(new BN(v, 16).umod(self.n), 32); };
  var f8 = function(v) { return be(new BN(v, 16).umod(n8), 32); };
  return pointsOut(this, native.mulAddBatch(CURVE.ed25519, pack(k1s, 32, f), pack(k2s, 32, f8), pack(p2s, 64, xy(32))), k1s.length, 32);
};
// curve.mont#mulBatch on curve25519: x-only points (mont.js:130-153); mulAdd throws in the reference and is left alone
elliptic.curve.mont.prototype.mulBatch = function mulBatch(points, ks) {
  var self = this;
  if (presetName(this) !== 'curve25519' || ks.some(function(k) { return new BN(k, 16).byteLength() > 32; }))
    return ks.map(function(k, i) { return points[i].mul(new BN(k, 16)); });
  init();
  var res = native.x25519Batch(pack(ks, 32, function(v) { return be(new BN(v, 16), 32); }),
    pack(points, 32, function(p) { return be(p.getX(), 32); }), 0);
  return ks.map(function(_, i) { return self.point(new BN(res.out.subarray(32 * i, 32 * i + 32)), new BN(1)); });
};

module.exports = elliptic;
