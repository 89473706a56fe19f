//! Raw FFI declarations for libaptb200.so (hand-written equivalent of what `bindgen include/aptb200.h`
//! emits).  SOURCE ONLY: there is no Rust toolchain in the image this repository is built and tested in,
//! so this file has never been compiled; the ABI it binds is exercised by the C++ and Python hosts.
#![allow(non_camel_case_types, dead_code)]

use std::os::raw::{c_char, c_float, c_int, c_void};

pub const APT_OK: c_int = 0;
pub const APT_ERR_RESAMPLE_TO_ZERO: c_int = 1;
pub const APT_ERR_TOO_SHORT: c_int = 2;
pub const APT_ERR_FEW_SYNC_FRAMES: c_int = 3;
pub const APT_ERR_WORK_RATE: c_int = 4;
pub const APT_ERR_RATE_OVERFLOW: c_int = 5;
pub const APT_ERR_CUDA: c_int = 6;
pub const APT_ERR_BAD_ARG: c_int = 7;
pub const APT_ERR_NOMEM: c_int = 8;
pub const APT_ERR_CAPACITY: c_int = 9;
pub const APT_ERR_EMPTY_RESULT: c_int = 10;

pub const APT_FILTER_NONE: c_int = 0;
pub const APT_FILTER_LOWPASS: c_int = 1;
pub const APT_FILTER_LOWPASS_DC: c_int = 2;

#[repr(C)]
#[derive(Clone, Copy, Debug)]
pub struct apt_settings {
    pub work_rate: u32,
    pub resample_atten: c_float,
    pub resample_delta_freq: c_float,
    pub resample_cutout: c_float,
    pub demodulation_atten: c_float,
}

#[repr(C)]
#[derive(Clone, Copy, Debug)]
pub struct apt_filter {
    pub kind: c_int,
    pub cutout_pi: c_float,
    pub atten: c_float,
    pub delta_w_pi: c_float,
}

pub type apt_status_cb = Option<unsafe extern "C" fn(progress: c_float, description: *const c_char, user: *mut c_void)>;

#[link(name = "aptb200")]
extern "C" {
    pub fn apt_strerror(status: c_int) -> *const c_char;
    pub fn apt_last_error() -> *const c_char;
    pub fn apt_filter_resample(f: *mut apt_filter, input_rate: u32, output_rate: u32);
    pub fn apt_filter_design(f: *const apt_filter, out: *mut c_float, cap: usize, n: *mut usize) -> c_int;
    pub fn apt_freq_hz(f_hz: c_float, rate_hz: u32) -> c_float;
    pub fn apt_resample_len(n: u64, input_rate: u32, output_rate: u32, f: *const apt_filter, nout: *mut u64) -> c_int;
    pub fn apt_resample_with_filter(signal: *const c_float, n: u64, input_rate: u32, output_rate: u32,
                                    f: *const apt_filter, out: *mut c_float, cap: u64, nout: *mut u64) -> c_int;
    pub fn apt_demodulate(signal: *const c_float, n: u64, carrier_pi: c_float, out: *mut c_float) -> c_int;
    pub fn apt_filter_signal(signal: *const c_float, n: u64, f: *const apt_filter, out: *mut c_float) -> c_int;
    pub fn apt_find_sync(signal: *const c_float, n: u64, work_rate: u32, positions: *mut u64, cap: usize,
                         npositions: *mut usize, corr: *mut c_float) -> c_int;
    pub fn apt_decode_len_bound(n: u64, input_rate: u32, s: *const apt_settings, bound: *mut u64) -> c_int;
    pub fn apt_decode(signal: *const c_float, n: u64, input_rate: u32, s: *const apt_settings, sync: c_int,
                      out: *mut c_float, cap: u64, nout: *mut u64, cb: apt_status_cb, user: *mut c_void) -> c_int;
    pub fn apt_decode_pcm16(pcm: *const i16, n: u64, input_rate: u32, s: *const apt_settings, sync: c_int,
                            out: *mut c_float, cap: u64, nout: *mut u64, cb: apt_status_cb, user: *mut c_void) -> c_int;
    pub fn apt_cache_clear();

    // WAV files and the resample tool (wav.rs, resample.rs)
    pub fn apt_wav_info_read(path: *const c_char, info: *mut apt_wav_info) -> c_int;
    pub fn apt_wav_load(path: *const c_char, out: *mut c_float, cap: u64, n: *mut u64, sample_rate: *mut u32) -> c_int;
    pub fn apt_wav_load_pcm16(path: *const c_char, out: *mut i16, cap: u64, n: *mut u64, sample_rate: *mut u32) -> c_int;
    pub fn apt_wav_write_i16(path: *const c_char, samples: *const i16, n: u64, sample_rate: u32) -> c_int;
    pub fn apt_quantize_i16(signal: *const c_float, n: u64, out: *mut i16) -> c_int;
    pub fn apt_resample_wav(input_path: *const c_char, output_path: *const c_char, output_rate: u32, atten: c_float,
                            delta_w_pi: c_float, nout: *mut u64) -> c_int;

    // image stage (front of noaa_apt::process)
    pub fn apt_decode_image_u8(signal: *const c_void, format: c_int, n: u64, input_rate: u32, s: *const apt_settings,
                               sync: c_int, contrast: c_int, percent: c_float, out: *mut u8, cap: u64, nout: *mut u64,
                               info: *mut apt_image_info, cb: apt_status_cb, user: *mut c_void) -> c_int;
    pub fn apt_map_signal_u8(signal: *const c_float, n: u64, low: c_float, high: c_float, out: *mut u8) -> c_int;
    pub fn apt_contrast_bounds(signal: *const c_float, n: u64, contrast: c_int, percent: c_float,
                               info: *mut apt_image_info) -> c_int;
    pub fn apt_telemetry_rows(signal: *const c_float, n: u64, mean_a: *mut c_float, mean_b: *mut c_float,
                              variance: *mut c_float) -> c_int;

    // the rest of noaa_apt::process (false colour, histogram equalisation, rotation), map overlay excepted
    pub fn apt_process(rows: *const c_float, n: u64, ps: *const apt_process_settings, out: *mut u8, cap: u64, nout: *mut u64,
                       info: *mut apt_image_info) -> c_int;
    pub fn apt_decode_image(signal: *const c_void, format: c_int, n: u64, input_rate: u32, s: *const apt_settings, sync: c_int,
                            ps: *const apt_process_settings, out: *mut u8, cap: u64, nout: *mut u64, info: *mut apt_image_info,
                            cb: apt_status_cb, user: *mut c_void) -> c_int;
    // live decoding (apt_stream_*): push audio as it arrives, get the rows that became final
    pub fn apt_stream_create(device: c_int, input_rate: u32, s: *const apt_settings, sync: c_int, max_push: u64,
                             st: *mut *mut apt_stream) -> c_int;
    pub fn apt_stream_destroy(st: *mut apt_stream);
    pub fn apt_stream_push_bound(st: *mut apt_stream, n: u64, cap_floats: *mut u64) -> c_int;
    pub fn apt_stream_push(st: *mut apt_stream, samples: *const c_void, format: c_int, n: u64, rows: *mut c_float, cap: u64,
                           nout: *mut u64) -> c_int;
    pub fn apt_stream_finish(st: *mut apt_stream, rows: *mut c_float, cap: u64, nout: *mut u64) -> c_int;
    pub fn apt_stream_reset(st: *mut apt_stream) -> c_int;
    pub fn apt_stream_sync_positions(st: *mut apt_stream, pos: *mut u64, cap: usize, n: *mut usize) -> c_int;
    pub fn apt_stream_get_info(st: *mut apt_stream, info: *mut apt_stream_info) -> c_int;
    pub fn apt_stream_geometry(input_rate: u32, s: *const apt_settings, sync: c_int, max_push: u64, info: *mut apt_stream_info) -> c_int;
    pub fn apt_iq_default_settings(iq_rate: u32, offset_hz: i32, s: *mut apt_iq_settings) -> c_int;
    pub fn apt_fm_demod_len(n: u64, s: *const apt_iq_settings, nout: *mut u64) -> c_int;
    pub fn apt_fm_demod(iq: *const c_void, format: c_int, n: u64, s: *const apt_iq_settings, out: *mut c_float, cap: u64,
                        nout: *mut u64) -> c_int;
    pub fn apt_decode_iq(iq: *const c_void, format: c_int, n: u64, s: *const apt_iq_settings, settings: *const apt_settings,
                         sync: c_int, out: *mut c_float, cap: u64, nout: *mut u64, cb: apt_status_cb, user: *mut c_void) -> c_int;
    pub fn apt_stream_create_iq(device: c_int, iq: *const apt_iq_settings, s: *const apt_settings, sync: c_int, max_push: u64,
                                st: *mut *mut apt_stream) -> c_int;
    pub fn apt_stream_geometry_iq(iq: *const apt_iq_settings, s: *const apt_settings, sync: c_int, max_push: u64,
                                  info: *mut apt_stream_info) -> c_int;
    pub fn apt_wav_load_iq16(path: *const c_char, out: *mut i16, cap: u64, n: *mut u64, sample_rate: *mut u32) -> c_int;
    // Finding the carriers of an I/Q recording (DESIGN.md §10, "Finding carriers")
    pub fn apt_iq_spectrum(iq: *const c_void, format: c_int, n: u64, iq_rate: u32, ss: *const apt_spectrum_settings,
                           psd: *mut c_float, cap: u64, nseg: *mut u32) -> c_int;
    pub fn apt_iq_find_carriers(iq: *const c_void, format: c_int, n: u64, s: *const apt_iq_settings,
                                cs: *const apt_carrier_search, out: *mut apt_carrier, cap: u32, count: *mut u32) -> c_int;
    pub fn apt_find_carriers_psd(psd: *const c_float, nfft: u32, iq_rate: u32, cutout: c_float, cs: *const apt_carrier_search,
                                 out: *mut apt_carrier, cap: u32, count: *mut u32) -> c_int;
    pub fn apt_decode_iq_channels(iq: *const c_void, format: c_int, n: u64, s: *const apt_iq_settings, offsets: *const i32,
                                  count: c_int, settings: *const apt_settings, sync: c_int, outs: *const *mut c_float,
                                  caps: *const u64, nouts: *mut u64, statuses: *mut c_int) -> c_int;
    pub fn apt_decode_iq_auto(iq: *const c_void, format: c_int, n: u64, s: *const apt_iq_settings,
                              cs: *const apt_carrier_search, settings: *const apt_settings, sync: c_int,
                              found: *mut apt_carrier, cap_found: u32, nfound: *mut u32, outs: *const *mut c_float,
                              caps: *const u64, nouts: *mut u64, statuses: *mut c_int) -> c_int;
    // PNG output: the file's bytes encoded on the device (DESIGN.md §11)
    pub fn apt_png_default_settings(ps: *mut apt_png_settings);
    pub fn apt_png_bound(width: u32, height: u32, channels: c_int, ps: *const apt_png_settings, bytes: *mut u64) -> c_int;
    pub fn apt_png_encode(pixels: *const u8, width: u32, height: u32, channels: c_int, ps: *const apt_png_settings,
                          out: *mut u8, cap: u64, nout: *mut u64) -> c_int;
    pub fn apt_decode_png(signal: *const c_void, format: c_int, n: u64, input_rate: u32, s: *const apt_settings, sync: c_int,
                          ps: *const apt_process_settings, png: *const apt_png_settings, out: *mut u8, cap: u64,
                          nout: *mut u64, info: *mut apt_image_info, cb: apt_status_cb, user: *mut c_void) -> c_int;
    pub fn apt_decode_batch_image(signals: *const *const c_void, format: c_int, lens: *const u64, count: c_int, input_rate: u32,
                                  s: *const apt_settings, sync: c_int, ps: *const apt_process_settings,
                                  png: *const apt_png_settings, outs: *const *mut u8, caps: *const u64, nouts: *mut u64,
                                  infos: *mut apt_image_info, statuses: *mut c_int, devices: *const c_int, ndevices: c_int,
                                  streams_per_device: c_int) -> c_int;
    pub fn apt_png_encode_batch(pixels: *const *const u8, heights: *const u32, count: u32, width: u32, channels: c_int,
                                ps: *const apt_png_settings, outs: *const *mut u8, caps: *const u64, nouts: *mut u64) -> c_int;
    pub fn apt_decoder_set_png_mode(dec: *mut apt_decoder, ps: *const apt_png_settings) -> c_int;
    pub fn apt_decoder_create(device: c_int, input_rate: u32, s: *const apt_settings, max_samples: u64,
                              dec: *mut *mut apt_decoder) -> c_int;
    pub fn apt_decoder_destroy(dec: *mut apt_decoder);
    pub fn apt_decoder_submit_host(dec: *mut apt_decoder, signal: *const c_void, format: c_int, n: u64, sync: c_int,
                                   out: *mut f32, cap: u64) -> c_int;
    pub fn apt_decoder_wait(dec: *mut apt_decoder, nout: *mut u64) -> c_int;
    pub fn apt_default_track_settings(ts: *mut apt_track_settings);
    pub fn apt_decoder_set_sync_mode(dec: *mut apt_decoder, mode: c_int, ts: *const apt_track_settings) -> c_int;
    pub fn apt_decode_wav_png(input_path: *const c_char, output_path: *const c_char, s: *const apt_settings, sync: c_int,
                              ps: *const apt_process_settings, png: *const apt_png_settings, info: *mut apt_image_info) -> c_int;
    // image output of a stream: the pass ends in its processed image or PNG file (DESIGN.md §9)
    pub fn apt_stream_set_process_mode(st: *mut apt_stream, ps: *const apt_process_settings, max_rows: u64) -> c_int;
    pub fn apt_stream_set_png_mode(st: *mut apt_stream, png: *const apt_png_settings) -> c_int;
    pub fn apt_stream_finish_image(st: *mut apt_stream, rows: *mut c_float, cap: u64, nout: *mut u64, image: *mut u8,
                                   image_cap: u64, image_n: *mut u64, info: *mut apt_image_info) -> c_int;
}

pub const APT_CU8: c_int = 2;
pub const APT_CF32: c_int = 3;
pub const APT_CS16: c_int = 4;

#[repr(C)]
#[derive(Clone, Copy, Debug, Default)]
pub struct apt_iq_settings {
    pub iq_rate: u32,
    pub audio_rate: u32,
    pub offset_hz: i32,
    pub cutout: c_float,
    pub delta_freq: c_float,
    pub atten: c_float,
}

#[repr(C)]
#[derive(Clone, Copy, Debug, Default)]
pub struct apt_spectrum_settings { pub nfft: u32, pub max_segments: u32 }

#[repr(C)]
#[derive(Clone, Copy, Debug, Default)]
pub struct apt_carrier_search { pub lo_hz: i32, pub hi_hz: i32, pub nfft: u32, pub max_segments: u32, pub min_snr_db: c_float }

#[repr(C)]
#[derive(Clone, Copy, Debug, Default)]
pub struct apt_carrier { pub offset_hz: i32, pub centre_hz: c_float, pub snr_db: c_float, pub apt_score: c_float, pub is_apt: c_int }

#[repr(C)]
pub struct apt_stream { _private: [u8; 0] }

#[repr(C)]
#[derive(Default, Clone, Copy)]
pub struct apt_stream_info { pub samples_in: u64, pub work_final: u64, pub rows_out: u64, pub peaks: u64, pub latency_work: u64,
                             pub max_push: u64, pub device_bytes: u64 }

pub const APT_F32: c_int = 0;
pub const APT_PCM16: c_int = 1;
pub const APT_CONTRAST_MINMAX: c_int = 0;
pub const APT_CONTRAST_PERCENT: c_int = 1;
pub const APT_CONTRAST_TELEMETRY: c_int = 2;
pub const APT_CONTRAST_HISTOGRAM: c_int = 3;
pub const APT_ERR_IO: c_int = 11;

#[repr(C)]
#[derive(Default, Clone, Copy)]
pub struct apt_wav_info { pub sample_rate: u32, pub channels: u32, pub bits_per_sample: u32, pub is_float: u32, pub frames: u64 }

#[repr(C)]
#[derive(Default, Clone, Copy)]
pub struct apt_image_info { pub low: f32, pub high: f32, pub rows: u64, pub telemetry_row: u64,
                            pub wedges_a: [f32; 16], pub wedges_b: [f32; 16] }

#[repr(C)]
#[derive(Clone, Copy)]
pub struct apt_process_settings { pub contrast: c_int, pub percent: c_float, pub rotate: c_int,
                                  pub palette: *const u8 /* 256*256*3 RGB or null */, pub tune: [c_float; 4], pub rgba: c_int }

#[repr(C)]
pub struct apt_decoder { _private: [u8; 0] }

#[repr(C)]
#[derive(Clone, Copy)]
pub struct apt_track_settings { pub delta: u32, pub lambda: f32 }
/// apt_sync_mode (apt_decoder_set_sync_mode)
pub const APT_SYNC_PEAKS: c_int = 0;
pub const APT_SYNC_TRACK: c_int = 1;

#[repr(C)]
#[derive(Clone, Copy)]
pub struct apt_png_settings { pub filter: c_int /* -1 adaptive, 0..4 fixed */, pub matches: c_int, pub block_bytes: u32,
                              pub rgb_from_rgba: c_int }

impl Default for apt_png_settings {
    fn default() -> Self { apt_png_settings { filter: -1, matches: 1, block_bytes: 65536, rgb_from_rgba: 0 } }
}

// Long recordings: finding the passes (DESIGN.md §12)
#[repr(C)]
#[derive(Default, Clone, Copy, Debug)]
pub struct apt_pass_search { pub enter: f32, pub exit: f32, pub max_gap_s: f32, pub min_length_s: f32 }   // 0: default

#[repr(C)]
#[derive(Default, Clone, Copy, Debug)]
pub struct apt_pass { pub start: u64, pub end: u64, pub first_window: u64, pub windows: u64, pub mean_quality: f32,
                      pub peak_quality: f32 }

#[repr(C)]
pub struct apt_recording { _private: [u8; 0] }

#[repr(C)]
#[derive(Default, Clone, Copy, Debug)]
pub struct apt_recording_info { pub samples: u64, pub work_samples: u64, pub windows: u64, pub device_bytes: u64,
                                pub input_rate: u32, pub row_samples: u32 }

#[link(name = "aptb200")]
extern "C" {
    pub fn apt_recording_create(device: c_int, signal: *const c_void, format: c_int, n: u64, input_rate: u32,
                                s: *const apt_settings, rec: *mut *mut apt_recording) -> c_int;
    pub fn apt_recording_destroy(rec: *mut apt_recording);
    pub fn apt_recording_get_info(rec: *mut apt_recording, info: *mut apt_recording_info) -> c_int;
    pub fn apt_recording_quality(rec: *mut apt_recording, q: *mut f32, cap: u64, nq: *mut u64) -> c_int;
    pub fn apt_find_passes_quality(q: *const f32, nq: u64, n: u64, input_rate: u32, ps: *const apt_pass_search,
                                   out: *mut apt_pass, cap: u32, count: *mut u32) -> c_int;
    pub fn apt_recording_decode(rec: *mut apt_recording, ranges: *const apt_pass, count: u32, sync: c_int,
                                ps: *const apt_process_settings, png: *const apt_png_settings, outs: *const *mut c_void,
                                caps: *const u64, nouts: *mut u64, infos: *mut apt_image_info, statuses: *mut c_int) -> c_int;
}

// Continuous feeds: watching for passes (DESIGN.md §13)
pub const APT_PASS_AOS: c_int = 1;
pub const APT_PASS_LOS: c_int = 2;
pub const APT_PASS_SEGMENT: c_int = 3;

#[repr(C)]
#[derive(Default, Clone, Copy, Debug)]
pub struct apt_pass_event { pub kind: c_int, pub window: u64, pub pass: apt_pass }

#[repr(C)]
pub struct apt_pass_tracker { _private: [u8; 0] }

#[repr(C)]
pub struct apt_watch { _private: [u8; 0] }

#[repr(C)]
#[derive(Clone, Copy)]
pub struct apt_watch_settings { pub sync: c_int, pub search: apt_pass_search, pub ps: *const apt_process_settings,
                                pub png: *const apt_png_settings, pub max_rows: u64, pub max_push: u64 }

#[repr(C)]
#[derive(Clone, Copy)]
pub struct apt_watch_event { pub ev: apt_pass_event, pub index: u32, pub status: c_int, pub rows: u64, pub info: apt_image_info,
                             pub data: *const c_void, pub bytes: u64 }

#[repr(C)]
#[derive(Default, Clone, Copy, Debug)]
pub struct apt_watch_info { pub samples_in: u64, pub segment_start: u64, pub windows: u64, pub passes: u64, pub open: u64,
                            pub device_bytes: u64, pub max_push: u64, pub latency_windows: u64 }

pub type apt_watch_cb = Option<unsafe extern "C" fn(ev: *const apt_watch_event, user: *mut c_void)>;
// One SDR's I/Q feed on several channels (DESIGN.md §14)
pub const APT_WATCH_IQ_MAX_CHANNELS: c_int = 8;
#[repr(C)]
pub struct apt_watch_iq { _private: [u8; 0] }
pub type apt_watch_iq_cb = Option<unsafe extern "C" fn(channel: c_int, ev: *const apt_watch_event, user: *mut c_void)>;

#[link(name = "aptb200")]
extern "C" {
    pub fn apt_pass_tracker_create(input_rate: u32, search: *const apt_pass_search, t: *mut *mut apt_pass_tracker) -> c_int;
    pub fn apt_pass_tracker_feed(t: *mut apt_pass_tracker, q: *const f32, nq: u64, events: *mut apt_pass_event, cap: u64,
                                 nev: *mut u64) -> c_int;
    pub fn apt_pass_tracker_finish(t: *mut apt_pass_tracker, n: u64, events: *mut apt_pass_event, cap: u64, nev: *mut u64) -> c_int;
    pub fn apt_pass_tracker_destroy(t: *mut apt_pass_tracker);
    pub fn apt_watch_create(device: c_int, input_rate: u32, s: *const apt_settings, ws: *const apt_watch_settings,
                            cb: apt_watch_cb, user: *mut c_void, w: *mut *mut apt_watch) -> c_int;
    pub fn apt_watch_geometry(input_rate: u32, s: *const apt_settings, ws: *const apt_watch_settings,
                              info: *mut apt_watch_info) -> c_int;
    pub fn apt_watch_push_bound(w: *mut apt_watch, n: u64, cap_q: *mut u64) -> c_int;
    pub fn apt_watch_push(w: *mut apt_watch, samples: *const c_void, format: c_int, n: u64, q: *mut f32, cap: u64,
                          nq: *mut u64) -> c_int;
    pub fn apt_watch_finish(w: *mut apt_watch, q: *mut f32, cap: u64, nq: *mut u64) -> c_int;
    pub fn apt_watch_reset(w: *mut apt_watch) -> c_int;
    pub fn apt_watch_get_info(w: *mut apt_watch, info: *mut apt_watch_info) -> c_int;
    pub fn apt_watch_destroy(w: *mut apt_watch);
    pub fn apt_fm_demod_channels(iq: *const c_void, format: c_int, n: u64, s: *const apt_iq_settings, offsets: *const i32,
                                 count: c_int, outs: *const *mut f32, cap: u64, nout: *mut u64) -> c_int;
    pub fn apt_watch_iq_geometry(iq: *const apt_iq_settings, offsets: *const i32, count: c_int, s: *const apt_settings,
                                 ws: *const apt_watch_settings, info: *mut apt_watch_info) -> c_int;
    pub fn apt_watch_iq_create(device: c_int, iq: *const apt_iq_settings, offsets: *const i32, count: c_int,
                               s: *const apt_settings, ws: *const apt_watch_settings, cb: apt_watch_iq_cb, user: *mut c_void,
                               w: *mut *mut apt_watch_iq) -> c_int;
    pub fn apt_watch_iq_push_bound(w: *mut apt_watch_iq, n: u64, cap_q: *mut u64) -> c_int;
    pub fn apt_watch_iq_push(w: *mut apt_watch_iq, iq: *const c_void, format: c_int, n: u64, q: *mut f32, cap: u64,
                             nq: *mut u64) -> c_int;
    pub fn apt_watch_iq_finish(w: *mut apt_watch_iq, q: *mut f32, cap: u64, nq: *mut u64) -> c_int;
    pub fn apt_watch_iq_reset(w: *mut apt_watch_iq) -> c_int;
    pub fn apt_watch_iq_get_info(w: *mut apt_watch_iq, channel: c_int, info: *mut apt_watch_info) -> c_int;
    pub fn apt_watch_iq_destroy(w: *mut apt_watch_iq);
}
