//! density-rs-shaped API over libdensity_b200.so (include/density_b200.h).
//!
//! Mirrors the reference's public surface for the accelerated path:
//!   * inherent `Chameleon::encode / decode` (src/algorithms/chameleon/chameleon.rs:45-53; cheetah.rs:57-65; lion.rs:74-82): a fresh
//!     dictionary per call -> the nine `extern "C"` symbols with the reference's own names;
//!   * `trait Codec` on an INSTANCE that is reused across calls (src/codec/codec.rs:12-127: `encode`, `decode`, `clear_state`,
//!     `safe_encode_buffer_size`, `block_size`, `decode_unit_size`, `signature_significant_bytes`) -> `density_b200_codec_*`.
//! Errors: the library returns 0 where the reference returns `Err` or panics (undersized buffer, truncated stream).

use std::ffi::{c_int, c_void};

#[derive(Debug)]
pub struct EncodeError {} // src/errors/encode_error.rs:4-13
#[derive(Debug)]
pub struct DecodeError {} // src/errors/decode_error.rs:4-13

#[repr(C)]
pub struct RawCodec {
    _private: [u8; 0],
}

unsafe extern "C" {
    // chameleon.rs:70-83, cheetah.rs:105-118, lion.rs:193-206
    pub fn chameleon_encode(input: *const u8, input_size: usize, output: *mut u8, output_size: usize) -> usize;
    pub fn chameleon_decode(input: *const u8, input_size: usize, output: *mut u8, output_size: usize) -> usize;
    pub fn chameleon_safe_encode_buffer_size(size: usize) -> usize;
    pub fn cheetah_encode(input: *const u8, input_size: usize, output: *mut u8, output_size: usize) -> usize;
    pub fn cheetah_decode(input: *const u8, input_size: usize, output: *mut u8, output_size: usize) -> usize;
    pub fn cheetah_safe_encode_buffer_size(size: usize) -> usize;
    pub fn lion_encode(input: *const u8, input_size: usize, output: *mut u8, output_size: usize) -> usize;
    pub fn lion_decode(input: *const u8, input_size: usize, output: *mut u8, output_size: usize) -> usize;
    pub fn lion_safe_encode_buffer_size(size: usize) -> usize;
    // device-resident, stream-ordered
    pub fn density_b200_encode_device(alg: c_int, d_in: *const u8, n: usize, d_out: *mut u8, cap: usize, d_out_size: *mut u64, stream: *mut c_void) -> c_int;
    pub fn density_b200_decode_device(alg: c_int, d_in: *const u8, n: usize, d_out: *mut u8, cap: usize, d_out_size: *mut u64, stream: *mut c_void) -> c_int;
    // the length a stream decodes to, without decoding it: {size, verdict} to d_result (device) / DENSITY_B200_OK with *out_size
    pub fn density_b200_decoded_size_device(alg: c_int, d_in: *const u8, n: usize, d_result: *mut u64, stream: *mut c_void) -> c_int;
    pub fn density_b200_decoded_size(alg: c_int, input: *const u8, n: usize, out_size: *mut u64) -> c_int;
    // bytes [first, first + len) of what a Chameleon stream decodes to: {written, size, verdict} to d_result (device) / *written
    pub fn density_b200_chameleon_decode_range_device(d_in: *const u8, n: usize, first: u64, len: u64, d_out: *mut u8, d_result: *mut u64, stream: *mut c_void) -> c_int;
    pub fn density_b200_chameleon_decode_range(input: *const u8, n: usize, first: u64, output: *mut u8, len: u64, written: *mut u64) -> c_int;
    // the Chameleon seek index: its length bound, its build, and a range decode that reads only the piece between two checkpoints
    pub fn density_b200_chameleon_index_bytes(n: usize, interval: u64) -> u64;
    pub fn density_b200_chameleon_index_build(input: *const u8, n: usize, interval: u64, index: *mut u8, index_cap: usize, index_len: *mut u64) -> c_int;
    pub fn density_b200_chameleon_decode_range_indexed(input: *const u8, n: usize, index: *const u8, index_len: usize, first: u64, output: *mut u8, len: u64, written: *mut u64) -> c_int;
    // a reused Codec instance (codec.rs:16,72,82)
    pub fn density_b200_codec_create(alg: c_int) -> *mut RawCodec;
    pub fn density_b200_codec_destroy(codec: *mut RawCodec);
    pub fn density_b200_codec_clear_state(codec: *mut RawCodec) -> c_int;
    pub fn density_b200_codec_encode(codec: *mut RawCodec, input: *const u8, input_size: usize, output: *mut u8, output_size: usize) -> usize;
    pub fn density_b200_codec_decode(codec: *mut RawCodec, input: *const u8, input_size: usize, output: *mut u8, output_size: usize) -> usize;
    pub fn density_b200_last_error() -> *const std::ffi::c_char;
}

/// src/codec/codec.rs:12-127, for the part of the trait the accelerated path implements.
pub trait Codec {
    fn block_size() -> usize;
    fn decode_unit_size() -> usize;
    fn signature_significant_bytes() -> usize;
    fn safe_encode_buffer_size(size: usize) -> usize;
    fn clear_state(&mut self);
    fn encode(&mut self, input: &[u8], output: &mut [u8]) -> Result<usize, EncodeError>;
    fn decode(&mut self, input: &[u8], output: &mut [u8]) -> Result<usize, DecodeError>;
}

macro_rules! algorithm {
    ($name:ident, $id:expr, $enc:ident, $dec:ident, $safe:ident, $block:expr, $unit:expr, $sig:expr) => {
        pub struct $name {
            raw: *mut RawCodec,
        }
        impl $name {
            /// `X::new()`: a zero-initialised dictionary (chameleon.rs:39-43).
            pub fn new() -> Self {
                let raw = unsafe { density_b200_codec_create($id) };
                assert!(!raw.is_null(), "density_b200_codec_create failed (no usable CUDA device?)");
                Self { raw }
            }
            /// The reference's inherent associated function: fresh state per call (chameleon.rs:45-48).
            pub fn encode(input: &[u8], output: &mut [u8]) -> Result<usize, EncodeError> {
                let n = unsafe { $enc(input.as_ptr(), input.len(), output.as_mut_ptr(), output.len()) };
                if n == 0 && !input.is_empty() { Err(EncodeError {}) } else { Ok(n) }
            }
            /// chameleon.rs:50-53
            pub fn decode(input: &[u8], output: &mut [u8]) -> Result<usize, DecodeError> {
                let n = unsafe { $dec(input.as_ptr(), input.len(), output.as_mut_ptr(), output.len()) };
                if n == 0 && !input.is_empty() { Err(DecodeError {}) } else { Ok(n) }
            }
            /// The output capacity `decode` needs for `input`: the bytes it decodes to, from the block boundaries without decoding.
            /// `Err` where `decode` fails at any capacity (a malformed stream) or the library could not run.
            pub fn decoded_size(input: &[u8]) -> Result<usize, DecodeError> {
                let mut size: u64 = 0;
                let rc = unsafe { density_b200_decoded_size($id, input.as_ptr(), input.len(), &mut size) };
                if rc == 0 { usize::try_from(size).map_err(|_| DecodeError {}) } else { Err(DecodeError {}) }
            }
        }
        impl Drop for $name {
            fn drop(&mut self) {
                unsafe { density_b200_codec_destroy(self.raw) }
            }
        }
        impl Codec for $name {
            fn block_size() -> usize { $block }
            fn decode_unit_size() -> usize { $unit }
            fn signature_significant_bytes() -> usize { $sig }
            fn safe_encode_buffer_size(size: usize) -> usize { unsafe { $safe(size) } }
            fn clear_state(&mut self) { unsafe { density_b200_codec_clear_state(self.raw); } }
            fn encode(&mut self, input: &[u8], output: &mut [u8]) -> Result<usize, EncodeError> {
                let n = unsafe { density_b200_codec_encode(self.raw, input.as_ptr(), input.len(), output.as_mut_ptr(), output.len()) };
                if n == 0 && !input.is_empty() { Err(EncodeError {}) } else { Ok(n) }
            }
            fn decode(&mut self, input: &[u8], output: &mut [u8]) -> Result<usize, DecodeError> {
                let n = unsafe { density_b200_codec_decode(self.raw, input.as_ptr(), input.len(), output.as_mut_ptr(), output.len()) };
                if n == 0 && !input.is_empty() { Err(DecodeError {}) } else { Ok(n) }
            }
        }
    };
}

algorithm!(Chameleon, 0, chameleon_encode, chameleon_decode, chameleon_safe_encode_buffer_size, 256, 8, 8); // chameleon.rs:138-147
algorithm!(Cheetah, 1, cheetah_encode, cheetah_decode, cheetah_safe_encode_buffer_size, 128, 4, 8); // cheetah.rs:188-197
algorithm!(Lion, 2, lion_encode, lion_decode, lion_safe_encode_buffer_size, 64, 4, 6); // lion.rs:317-326

impl Chameleon {
    /// Bytes `[first, first + output.len())` of what `input` decodes to, without decoding the bytes in front of them: the bytes written,
    /// `min(first + output.len(), S) - first`, or 0 when `first >= S` (S: the decoded size). `Err` where `decode` fails at any capacity
    /// (a malformed stream) or the library could not run.
    pub fn decode_range(input: &[u8], first: u64, output: &mut [u8]) -> Result<usize, DecodeError> {
        let mut written: u64 = 0;
        let rc = unsafe {
            density_b200_chameleon_decode_range(input.as_ptr(), input.len(), first, output.as_mut_ptr(), output.len() as u64, &mut written)
        };
        if rc == 0 { usize::try_from(written).map_err(|_| DecodeError {}) } else { Err(DecodeError {}) }
    }

    /// The seek index of `input` with a checkpoint every `interval` decoded bytes (a positive multiple of 256): a byte blob that can be
    /// stored beside the stream. `Err` on a malformed stream, a bad interval, or when the library could not run.
    pub fn build_index(input: &[u8], interval: u64) -> Result<Vec<u8>, DecodeError> {
        let bound = unsafe { density_b200_chameleon_index_bytes(input.len(), interval) };
        let mut index = vec![0u8; usize::try_from(bound).map_err(|_| DecodeError {})?];
        if index.is_empty() {
            return Err(DecodeError {});
        }
        let mut len: u64 = 0;
        let rc = unsafe { density_b200_chameleon_index_build(input.as_ptr(), input.len(), interval, index.as_mut_ptr(), index.len(), &mut len) };
        if rc != 0 {
            return Err(DecodeError {});
        }
        index.truncate(len as usize);
        Ok(index)
    }

    /// `decode_range` from the seek index `build_index` returned for `input`: only the stream between the two checkpoints around the
    /// window is read and decoded. `Err` as `decode_range`, and when the index does not describe `input`.
    pub fn decode_range_indexed(input: &[u8], index: &[u8], first: u64, output: &mut [u8]) -> Result<usize, DecodeError> {
        let mut written: u64 = 0;
        let rc = unsafe {
            density_b200_chameleon_decode_range_indexed(input.as_ptr(), input.len(), index.as_ptr(), index.len(), first, output.as_mut_ptr(),
                                                        output.len() as u64, &mut written)
        };
        if rc == 0 { usize::try_from(written).map_err(|_| DecodeError {}) } else { Err(DecodeError {}) }
    }
}

#[cfg(test)]
mod tests {
    // the reference's own known-answer test (src/lib.rs:19-41), through this binding
    use super::*;
    const TEST_DATA: &str = "testtesttesttesttesttesttesttesttesttesttesttesttesttesttesttesttesttesttesttesttesttesttesttesttesttesttesttesttesttesttestt";
    #[test]
    fn chameleon() {
        let mut out = vec![0u8; TEST_DATA.len()];
        let n = Chameleon::encode(TEST_DATA.as_bytes(), &mut out).unwrap();
        assert_eq!(&out[0..12], &[0xfe, 0xff, 0xff, 0x7f, 0, 0, 0, 0, b't', b'e', b's', b't']);
        let mut dec = vec![0u8; TEST_DATA.len()];
        let m = Chameleon::decode(&out[0..n], &mut dec).unwrap();
        assert_eq!(&dec[0..m], TEST_DATA.as_bytes());
    }
}
