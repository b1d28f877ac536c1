"""What a stream decodes to, and whether it is malformed, from two independent sources (numpy and the oracle only).

`oracle_size(alg, stream)`: the oracle's decode at a capacity no stream can reach. A non-zero result is the size, verdict 0. A zero result
is either a malformed stream (the decoder reads past its end) or one of the few streams that decode to nothing: the empty stream, and a
stream that is exactly one signature whose first flag is PLAIN (codec.rs:102-123: no main-loop block fits, the first unit of the tail
is partial, and its PLAIN flag meets 0 bytes left, which ends the stream). Any other stream writes at least one byte or fails, so that
rule separates the two.

`model_size(alg, stream)`: the main loop from synth_streams.walk, then the tail loop's control flow (codec.rs:102-123 with
chameleon.rs:116-135, cheetah.rs:165-185, lion.rs:291-314) walked in Python, counting bytes and reads past the end. It does not decode
a single quad.

Both return (size, verdict), verdict 0 or MALFORMED (then size 0); tests/test_decoded_size_cpu.py checks that they agree.
"""
import numpy as np

import oracle
import synth_streams as ss

MALFORMED = 3                                       # DENSITY_B200_EMALFORMED
UNIT = {"chameleon": 8, "cheetah": 4, "lion": 4}    # decode_unit_size (chameleon.rs:142, cheetah.rs:191, lion.rs:320)


def _first_flag(alg, stream):
    return int(stream[0]) & ((1 << ss.FB[alg]) - 1)


def oracle_cap(n):
    """more than any n-byte stream decodes to (the largest ratio is a Cheetah block of 32 predicted quads: 8 bytes -> 128)"""
    return 16 * n + 256


def oracle_size(alg, stream):
    s = np.asarray(stream, np.uint8)
    n = s.size
    r = oracle.decode(alg, s, oracle_cap(n)).size if n else 0
    if r:
        return r, 0
    empty = n == 0 or (n == ss.SIG[alg] and _first_flag(alg, s) == 0)
    return (0, 0) if empty else (0, MALFORMED)


def _payload(alg, flag):
    return ss.PAYLOAD[alg][flag]


def model_size(alg, stream):
    s = np.asarray(stream, np.uint8)
    n, bs, sb, fb, unit = s.size, ss.BS[alg], ss.SIG[alg], ss.FB[alg], UNIT[alg]
    w = ss.walk(alg, s)
    ps = ss._Prot(*w["state"])
    idx, out = w["tail_off"], w["main_blocks"] * bs
    buf = s.tobytes()
    while n - idx > 0:
        if ps.step_copy():                                  # codec.rs:104-110
            if n - idx > bs:
                idx += bs; out += bs
                continue
            out += n - idx
            break
        mark = idx
        if n - idx < sb:
            return 0, MALFORMED
        sig = int.from_bytes(buf[idx:idx + sb], "little")
        idx += sb
        end = False
        for _ in range(bs // unit):
            partial = n - idx < unit                        # decode_partial_unit for the whole unit
            for _ in range(unit // 4):
                f = sig & ((1 << fb) - 1)
                sig >>= fb
                if partial and f == 0 and n - idx < 4:      # the last 0-3 bytes, raw, and the stream ends
                    out += n - idx; idx = n
                    end = True
                    break
                k = _payload(alg, f)
                if n - idx < k:
                    return 0, MALFORMED
                idx += k; out += 4
            if end:
                break
        if end:
            break
        ps.step_update(idx - mark >= bs)
    return out, 0
