"""Argument coercion of the reference's L1 stream layer (lib/Util.js:9-101, lib/Stream.js).

``input``  : object with ``readByte()`` (drained until it returns -1, Stream.EOF lib/Stream.js:4)
             or any bytes-like / sequence of ints.
``output`` : object with ``writeByte(b)`` -> every byte is pushed to it and IT is returned;
             an ``int`` -> exact-size result, ``TypeError('outputsize does not match decoded input')``
             if the result does not fill it exactly (lib/Util.js:69-71, 90-92);
             a writable buffer (bytearray / numpy uint8) -> filled in place under the same rule;
             ``None`` -> a fresh ``bytes`` object (the reference returns a trimmed Uint8Array).
On a failed decode the output gets the bytes decoded before the error (``partial=True``), as the reference's output
stream has them when it throws: a stream receives them all, a buffer has its first min(len(data), len(buffer)) bytes
overwritten (a typed array drops writes past its end) and the rest left alone; a size or ``None`` shows nothing.
"""
import numpy as np

EOF_BYTE = -1


def coerce_input(inp):
    if hasattr(inp, "readByte"):
        out = bytearray()
        while True:
            b = inp.readByte()
            if b == EOF_BYTE or b is None:
                break
            out.append(b & 0xFF)
        return np.frombuffer(bytes(out), dtype=np.uint8)
    if isinstance(inp, np.ndarray):
        return np.ascontiguousarray(inp, dtype=np.uint8).ravel()
    if isinstance(inp, (bytes, bytearray, memoryview)):
        return np.frombuffer(inp, dtype=np.uint8)
    return np.array(list(inp), dtype=np.uint8)


def deliver_output(output, data, partial=False):
    """data: numpy uint8 view of the result (of the prefix in front of a decode error when `partial`).  Implements
    coerceOutputStream + retval."""
    if output is None:
        return data.tobytes()
    if hasattr(output, "writeByte"):
        for b in data.tobytes():
            output.writeByte(b)
        return output
    if partial:
        # nothing is observable of a size or of an output the success path would reject: the decode error stands alone
        if not isinstance(output, (bool, int)):
            try:
                mv = memoryview(output).cast("B")
                k = min(mv.nbytes, data.size)
                mv[:k] = data[:k].tobytes()
            except TypeError:
                pass
        return output
    if isinstance(output, bool):
        raise TypeError("output must be a stream, a size or a buffer")
    if isinstance(output, int):
        if output != data.size:
            raise TypeError("outputsize does not match decoded input")
        return data.tobytes()
    mv = memoryview(output)
    if mv.nbytes != data.size:
        raise TypeError("outputsize does not match decoded input")
    mv.cast("B")[:] = data.tobytes()
    return output
