// index.js -- JavaScript shim with the export names of compressjs' main.js for the bzip2 path.
// Argument coercion (streams / buffers / sizes) stays in JavaScript exactly as the reference does it;
// the per-block work goes to the N-API addon (addon.cc -> libb2bz.so -> CUDA).
'use strict';
var native = require('./build/Release/b2bz.node');

var EOF = -1;
function drain(input) {                       // Util.coerceInputStream semantics
  if (input && typeof input.readByte === 'function') {
    var bytes = [], b;
    while ((b = input.readByte()) !== EOF) { bytes.push(b); }
    return Buffer.from(bytes);
  }
  return Buffer.isBuffer(input) ? input : Buffer.from(input);
}
// partial: data is what a failed decode had written; a stream gets all of it, a buffer what fits (a typed array drops
// writes past its end), a size nothing, as the reference's output stream when it throws
function deliver(output, data, partial) {     // Util.coerceOutputStream + retval semantics
  if (output && typeof output === 'object' && typeof output.writeByte === 'function') {
    for (var i = 0; i < data.length; i++) { output.writeByte(data[i]); }
    return output;
  }
  if (typeof output === 'number') {
    if (partial) { return output; }
    if (output !== data.length) { throw new TypeError('outputsize does not match decoded input'); }
    return new Uint8Array(data);
  }
  if (output) {
    if (!partial && output.length !== data.length) { throw new TypeError('outputsize does not match decoded input'); }
    for (var j = 0; j < data.length && j < output.length; j++) { output[j] = data[j]; }
    return output;
  }
  return new Uint8Array(data);
}
// a decode whose error carries the bytes decoded before it (addon.cc): deliver those, then rethrow
function decode(output, call) {
  var data;
  try { data = call(); } catch (e) {
    if (e.partial) { deliver(output, e.partial, true); }
    throw e;
  }
  return deliver(output, data);
}

var Bzip2 = Object.create(null);
// options.flavor: 'compressjs' (the default) or 'libbz2': compressFile writes the bytes bzip2 -N writes, decompressFile
// reads as bzip2 -d reads (include/b2bz.h B2_BZ2_LIBBZ2)
var FLAVORS = { compressjs: 0, libbz2: 1 };
function flavor(options) {
  var name = (options && options.flavor !== undefined) ? options.flavor : 'compressjs';
  if (!Object.prototype.hasOwnProperty.call(FLAVORS, name)) { throw new Error('unknown bzip2 flavor ' + name); }
  return FLAVORS[name];
}
Bzip2.compressFile = function(inStream, outStream, props, options) {
  var fl = flavor(options);
  var level = (typeof props === 'number') ? props : 9;
  if (level < 1 || level > 9) { throw new Error('Invalid block size multiplier'); }
  return deliver(outStream, native.compressFile(drain(inStream), level, fl));
};
Bzip2.decompressFile = function(input, output, multistream, options) {
  var fl = flavor(options);   // before anything is read
  var data = drain(input);
  return decode(output, function() { return native.decompressFile(data, !!multistream, fl); });
};
Bzip2.decompressBlock = function(input, pos, output) {
  var data = drain(input);
  return decode(output, function() { return native.decompressBlock(data, pos); });
};
// GPU extension: decompressBlock at every position, in one pass.  No output: an array of Uint8Arrays, one per position;
// a writeByte stream receives every position's bytes in order (on an error, what the per-position loop would have
// written) and is returned.  A size or a buffer has no meaning for several blocks.
Bzip2.decompressBlocks = function(input, positions, output) {
  var stream = !!output && typeof output === 'object' && typeof output.writeByte === 'function';
  if (output !== undefined && output !== null && !stream) {
    throw new TypeError('decompressBlocks writes to a stream or returns an array');
  }
  var data = drain(input), r;
  try { r = native.decompressBlocks(data, Float64Array.from(positions)); } catch (e) {
    if (stream && e.partial) { deliver(output, e.partial, true); }
    throw e;
  }
  if (stream) { return deliver(output, r[0]); }
  var blocks = [], s = 0;
  r[1].forEach(function(e) { blocks.push(new Uint8Array(r[0].subarray(s, e))); s = e; });
  return blocks;
};
// GPU extension: the intact blocks of a damaged file (include/b2bz.h b2_bzip2_recover).  Returns [output, blocks]:
// output gets the intact blocks' bytes, or with opts.repair one bzip2 stream of them; blocks has one row per block magic,
// its status a string.
var REC_STATUS = ['INTACT', 'BAD_CRC', 'DATA_ERROR', 'OBSOLETE', 'INSIDE'];
Bzip2.recover = function(input, output, opts) {
  var r = native.recover(drain(input), !!(opts && opts.repair));
  var blocks = r[1].map(function(b) {
    return {bitpos: b[0], endbit: b[1], out_off: b[2], size: b[3], crc: b[4], got: b[5], status: REC_STATUS[b[6]]};
  });
  return [deliver(output, r[0]), blocks];
};
Bzip2.table = function(input, callback, multistream) {
  var rows;
  try { rows = native.table(drain(input), !!multistream); } catch (e) {
    (e.rows || []).forEach(function(r) { callback(r[0], r[1]); });
    throw e;
  }
  rows.forEach(function(r) { callback(r[0], r[1]); });
};

var BWT = Object.create(null);
BWT.bwtransform2 = function(T, U, n) { return native.bwtransform2(T, U, n); };
// the sentinel family (lib/BWT.js:305-363); the reference's scratch arrays A / LF are accepted and ignored
BWT.suffixsort = function(T, SA, n) { return native.suffixsort(T, SA, n); };
BWT.bwtransform = function(T, U, A, n) { return native.bwtransform(T, U, n); };
BWT.unbwtransform = function(T, U, LF, n, pidx) { native.unbwtransform(T, U, n, pidx); };

var BWTC = Object.create(null);   // lib/BWTC.js:10-231
BWTC.MAGIC = 'bwtc';
BWTC.compressFile = function(inStream, outStream, props) {
  var level = (typeof props === 'number' && props >= 1 && props <= 9) ? props : 9;   // :16-19
  return deliver(outStream, native.bwtcCompressFile(drain(inStream), level));
};
BWTC.decompressFile = function(input, output) {
  return deliver(output, native.bwtcDecompressFile(drain(input)));
};

module.exports = Object.freeze({ version: '0.0.1', Bzip2: Bzip2, BWT: BWT, BWTC: BWTC });
