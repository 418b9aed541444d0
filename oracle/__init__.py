"""CPU oracle for the Curvine sequential block-read hot path.

TEST INFRASTRUCTURE ONLY.  Nothing under ``oracle/`` is part of the product:
only ``tests/``, ``__graft_entry__.smoke()`` and ``bench.py``'s CPU-baseline /
``--impl reference`` legs may import, link or execute it (plus the measurement
scripts ``tools/c3_ssd_tier.py`` / ``tools/c5_smallfiles.py``, which time its CPU
reader beside the GPU path exactly as bench.py's CPU-baseline leg does), and there
only as the checker (or as the timed CPU baseline), never as the thing shipped.

It is a *restatement* of the reference's algorithm for this path, written from
the reference sources cited function by function (paths relative to the
CurvineIO/curvine source tree).  The reference is Rust (905 crates, not
vendored), so no binary of it is built beside the oracle.

Pinning status (SURVEY.md §8c):
  * wire status byte  -- pinned by the reference's only known-answer test,
    ``orpc/tests/common_test.rs:18-30`` (``Status(Running, Error).encode() == 19``).
  * CRC-32 (ISO-HDLC) -- the reference calls ``crc32fast::hash`` (crates.io,
    pin 1.4.2 / lock 1.5.0, not vendored; call site ``orpc/src/common/utils.rs:73-75``).
    Pinned here to the published check value 0xCBF43926 and to ``zlib.crc32``;
    the reference's own tests only assert write-side == read-side sums
    ("parity unpinned" for absolute CRC values inside the reference itself).
  * CRC-32C           -- absent from the reference (north_star's addition);
    pinned to the published check value 0xE3069283 and a bitwise implementation.
  * frame bytes       -- the reference holds no golden frame dump: "parity
    unpinned" beyond the status nibble; vectors in tests/golden are derived from
    the codec source and checked by encode->decode round trips and the
    ``total_len = 18 + header_len + data_len`` identity (rpc_message.rs:305,329).
  * index math        -- pinned by ``fs_reader_parallel.rs:194-220``,
    ``read_detector.rs:242-528`` and ``inode_id.rs:100-118`` (restated in tests/).
"""
