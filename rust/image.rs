//! Optional fast paths for `noaa_apt::process` (noaa_apt.rs:132-240).  `decode_to_gray`: decode + contrast bounds +
//! `map_signal_u8` in one library call, so that the rows leave the GPU as u8.  `decode_to_image`: decode + the whole of
//! `process` but the map overlay -- false colour, grey histogram equalisation and `Rotate::Yes` run on the device and only
//! the RGBA pixels cross PCIe.  `decode_to_png`: the same, then the PNG encoding on the device, so that only the file's
//! bytes cross PCIe and `img.save` (main.rs:115) becomes a plain write.  SOURCE ONLY (no Rust toolchain in the image this repository is built in).  The map
//! overlay, the orbit behind `Rotate::Orbit` and colour histogram equalisation (Lab) stay in Rust.

use std::os::raw::c_void;

use crate::aptb200_sys as sys;
use crate::config;
use crate::context::Context;
use crate::decode::to_error;
use crate::dsp::{Rate, Signal};
use crate::err;
use crate::noaa_apt::{ColorSettings, Contrast, Rotate};

/// (GrayImage bytes of width PX_PER_ROW, contrast bounds) for the three contrast modes the library implements.
pub fn decode_to_gray(
    context: &mut Context,
    settings: &config::Settings,
    signal: &Signal,
    input_rate: Rate,
    sync: bool,
    contrast: &Contrast,
) -> err::Result<(Vec<u8>, f32, f32)> {
    let (mode, percent) = match contrast {
        Contrast::MinMax => (sys::APT_CONTRAST_MINMAX, 0.0f32),
        Contrast::Percent(p) => (sys::APT_CONTRAST_PERCENT, *p),
        Contrast::Telemetry => (sys::APT_CONTRAST_TELEMETRY, 0.0f32),
        Contrast::Histogram => return Err(err::Error::FeatureNotAvailable(vec!["device histogram equalisation".into()])),
    };
    let s = sys::apt_settings::from(settings);
    let mut bound = 0u64;
    let st = unsafe { sys::apt_decode_len_bound(signal.len() as u64, input_rate.get_hz(), &s, &mut bound) };
    if st != 0 { return Err(to_error(st)); }
    let mut out = vec![0u8; bound.max(1) as usize];
    let mut n = 0u64;
    let mut info = sys::apt_image_info::default();
    let st = unsafe {
        sys::apt_decode_image_u8(signal.as_ptr() as *const c_void, sys::APT_F32, signal.len() as u64, input_rate.get_hz(), &s,
                                 sync as i32, mode, percent, out.as_mut_ptr(), out.len() as u64, &mut n, &mut info,
                                 Some(crate::decode::status_trampoline), context as *mut _ as *mut c_void)
    };
    if st != 0 { return Err(to_error(st)); }
    out.truncate(n as usize);
    Ok((out, info.low, info.high))
}

/// The RGBA bytes (width PX_PER_ROW, 4 bytes per pixel) `process` returns without a map overlay, for
/// `Contrast::{MinMax, Percent, Telemetry, Histogram}` x false colour x `Rotate::{No, Yes}`.  `Rotate::Orbit` is resolved
/// by the caller with `processing::south_to_north_pass` and passed as `Rotate::Yes` or `Rotate::No`.  The palette is
/// loaded here as `processing::false_color` loads it (processing.rs:110-116).
pub fn decode_to_image(
    context: &mut Context,
    settings: &config::Settings,
    signal: &Signal,
    input_rate: Rate,
    sync: bool,
    contrast: &Contrast,
    rotate: &Rotate,
    color: Option<&ColorSettings>,
) -> err::Result<(Vec<u8>, f32, f32)> {
    let (mode, percent) = match contrast {
        Contrast::MinMax => (sys::APT_CONTRAST_MINMAX, 0.0f32),
        Contrast::Percent(p) => (sys::APT_CONTRAST_PERCENT, *p),
        Contrast::Telemetry => (sys::APT_CONTRAST_TELEMETRY, 0.0f32),
        Contrast::Histogram => (sys::APT_CONTRAST_HISTOGRAM, 0.0f32),
    };
    if color.is_some() && mode == sys::APT_CONTRAST_HISTOGRAM {
        return Err(err::Error::FeatureNotAvailable(vec!["device colour histogram equalisation".into()]));
    }
    let rotate = match rotate {
        Rotate::Yes => 1,
        Rotate::No => 0,
        Rotate::Orbit => return Err(err::Error::InvalidInput("resolve Rotate::Orbit before decode_to_image".into())),
    };
    let palette = match color {
        Some(c) => {
            let p = ::image::open(&c.palette_filename)
                .map_err(|_| err::Error::InvalidInput(format!("Could not load {:?}", &c.palette_filename)))?
                .into_rgb8();
            if p.width() != 256 || p.height() != 256 {
                return Err(err::Error::InvalidInput("Invalid palette image dimensions".to_string()));
            }
            Some(p.into_raw())
        }
        None => None,
    };
    let tune = color.map_or([0.0f32; 4], |c| [c.ch_a_tune_start, c.ch_a_tune_end, c.ch_b_tune_start, c.ch_b_tune_end]);
    let ps = sys::apt_process_settings {
        contrast: mode,
        percent,
        rotate,
        palette: palette.as_ref().map_or(std::ptr::null(), |p| p.as_ptr()),
        tune,
        rgba: 1,
    };
    let s = sys::apt_settings::from(settings);
    let mut bound = 0u64;
    let st = unsafe { sys::apt_decode_len_bound(signal.len() as u64, input_rate.get_hz(), &s, &mut bound) };
    if st != 0 { return Err(to_error(st)); }
    let mut out = vec![0u8; (bound * 4).max(1) as usize];
    let mut n = 0u64;
    let mut info = sys::apt_image_info::default();
    let st = unsafe {
        sys::apt_decode_image(signal.as_ptr() as *const c_void, sys::APT_F32, signal.len() as u64, input_rate.get_hz(), &s,
                              sync as i32, &ps, out.as_mut_ptr(), out.len() as u64, &mut n, &mut info,
                              Some(crate::decode::status_trampoline), context as *mut _ as *mut c_void)
    };
    if st != 0 { return Err(to_error(st)); }
    out.truncate(n as usize);
    Ok((out, info.low, info.high))
}

/// The PNG file (bytes to write as they are) of what `decode_to_image` returns, encoded on the device (DESIGN.md §11).
/// Without a map overlay this replaces `img.save(&output_filename)` (main.rs:115).  With a map, call `decode_to_image`,
/// run `map::draw_map` on the RGBA and encode with `encode_png`.
pub fn decode_to_png(
    context: &mut Context,
    settings: &config::Settings,
    signal: &Signal,
    input_rate: Rate,
    sync: bool,
    contrast: &Contrast,
    rotate: &Rotate,
    color: Option<&ColorSettings>,
) -> err::Result<(Vec<u8>, f32, f32)> {
    let (mode, percent) = match contrast {
        Contrast::MinMax => (sys::APT_CONTRAST_MINMAX, 0.0f32),
        Contrast::Percent(p) => (sys::APT_CONTRAST_PERCENT, *p),
        Contrast::Telemetry => (sys::APT_CONTRAST_TELEMETRY, 0.0f32),
        Contrast::Histogram => (sys::APT_CONTRAST_HISTOGRAM, 0.0f32),
    };
    if color.is_some() && mode == sys::APT_CONTRAST_HISTOGRAM {
        return Err(err::Error::FeatureNotAvailable(vec!["device colour histogram equalisation".into()]));
    }
    let rotate = match rotate {
        Rotate::Yes => 1,
        Rotate::No => 0,
        Rotate::Orbit => return Err(err::Error::InvalidInput("resolve Rotate::Orbit before decode_to_png".into())),
    };
    let palette = match color {
        Some(c) => {
            let p = ::image::open(&c.palette_filename)
                .map_err(|_| err::Error::InvalidInput(format!("Could not load {:?}", &c.palette_filename)))?
                .into_rgb8();
            if p.width() != 256 || p.height() != 256 {
                return Err(err::Error::InvalidInput("Invalid palette image dimensions".to_string()));
            }
            Some(p.into_raw())
        }
        None => None,
    };
    let tune = color.map_or([0.0f32; 4], |c| [c.ch_a_tune_start, c.ch_a_tune_end, c.ch_b_tune_start, c.ch_b_tune_end]);
    let ps = sys::apt_process_settings {
        contrast: mode,
        percent,
        rotate,
        palette: palette.as_ref().map_or(std::ptr::null(), |p| p.as_ptr()),
        tune,
        rgba: 1,
    };
    let png = sys::apt_png_settings::default();
    let s = sys::apt_settings::from(settings);
    let mut bound = 0u64;
    let st = unsafe { sys::apt_decode_len_bound(signal.len() as u64, input_rate.get_hz(), &s, &mut bound) };
    if st != 0 { return Err(to_error(st)); }
    let rows = (bound / crate::decode::PX_PER_ROW as u64).max(1);
    let mut cap = 0u64;
    let st = unsafe { sys::apt_png_bound(crate::decode::PX_PER_ROW as u32, rows as u32, 4, &png, &mut cap) };
    if st != 0 { return Err(to_error(st)); }
    let mut out = vec![0u8; cap as usize];
    let mut n = 0u64;
    let mut info = sys::apt_image_info::default();
    let st = unsafe {
        sys::apt_decode_png(signal.as_ptr() as *const c_void, sys::APT_F32, signal.len() as u64, input_rate.get_hz(), &s,
                            sync as i32, &ps, &png, out.as_mut_ptr(), out.len() as u64, &mut n, &mut info,
                            Some(crate::decode::status_trampoline), context as *mut _ as *mut c_void)
    };
    if st != 0 { return Err(to_error(st)); }
    out.truncate(n as usize);
    Ok((out, info.low, info.high))
}

/// PNG bytes of RGBA pixels (width PX_PER_ROW), e.g. after `map::draw_map`, encoded on the device.
pub fn encode_png(rgba: &[u8], width: u32) -> err::Result<Vec<u8>> {
    let height = (rgba.len() / (4 * width as usize)) as u32;
    let png = sys::apt_png_settings::default();
    let mut cap = 0u64;
    let st = unsafe { sys::apt_png_bound(width, height, 4, &png, &mut cap) };
    if st != 0 { return Err(to_error(st)); }
    let mut out = vec![0u8; cap as usize];
    let mut n = 0u64;
    let st = unsafe { sys::apt_png_encode(rgba.as_ptr(), width, height, 4, &png, out.as_mut_ptr(), cap, &mut n) };
    if st != 0 { return Err(to_error(st)); }
    out.truncate(n as usize);
    Ok(out)
}
