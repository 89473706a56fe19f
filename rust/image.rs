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
    let (mode, percent, rotate, palette, tune) = png_process_parts(contrast, rotate, color)?;
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

/// The apt_process_settings parts of the PNG entry points: contrast mode and percent, rotation, the palette's RGB bytes
/// (kept alive by the caller) and the tune values.
pub(crate) fn png_process_parts(
    contrast: &Contrast,
    rotate: &Rotate,
    color: Option<&ColorSettings>,
) -> err::Result<(i32, f32, i32, Option<Vec<u8>>, [f32; 4])> {
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
        Rotate::Orbit => return Err(err::Error::InvalidInput("resolve Rotate::Orbit before decoding to PNG".into())),
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
    Ok((mode, percent, rotate, palette, tune))
}

/// `decode_to_png` of every recording of a batch, sharded over `devices` (recording i -> devices[i % len]) as
/// `apt_decode_batch` does; the images of each device are encoded together on the device.  Per recording: the PNG bytes
/// and contrast bounds, or the error of that recording alone.
pub fn decode_batch_to_png(
    settings: &config::Settings,
    signals: &[Signal],
    input_rate: Rate,
    sync: bool,
    contrast: &Contrast,
    rotate: &Rotate,
    color: Option<&ColorSettings>,
    devices: &[i32],
    streams_per_device: i32,
) -> err::Result<Vec<err::Result<(Vec<u8>, f32, f32)>>> {
    let (mode, percent, rotate, palette, tune) = png_process_parts(contrast, rotate, color)?;
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
    let count = signals.len();
    let mut outs: Vec<Vec<u8>> = Vec::with_capacity(count);
    for signal in signals {
        let mut bound = 0u64;
        let st = unsafe { sys::apt_decode_len_bound(signal.len() as u64, input_rate.get_hz(), &s, &mut bound) };
        if st != 0 { return Err(to_error(st)); }
        let rows = (bound / crate::decode::PX_PER_ROW as u64).max(1);
        let mut cap = 0u64;
        let st = unsafe { sys::apt_png_bound(crate::decode::PX_PER_ROW as u32, rows as u32, 4, &png, &mut cap) };
        if st != 0 { return Err(to_error(st)); }
        outs.push(vec![0u8; cap as usize]);
    }
    let sigs: Vec<*const c_void> = signals.iter().map(|x| x.as_ptr() as *const c_void).collect();
    let lens: Vec<u64> = signals.iter().map(|x| x.len() as u64).collect();
    let caps: Vec<u64> = outs.iter().map(|o| o.len() as u64).collect();
    let ptrs: Vec<*mut u8> = outs.iter_mut().map(|o| o.as_mut_ptr()).collect();
    let mut nouts = vec![0u64; count];
    let mut infos = vec![sys::apt_image_info::default(); count];
    let mut statuses = vec![-1i32; count];   // -1: not written (never "ok" unless the library says so)
    let st = unsafe {
        sys::apt_decode_batch_image(sigs.as_ptr(), sys::APT_F32, lens.as_ptr(), count as i32, input_rate.get_hz(), &s,
                                    sync as i32, &ps, &png, ptrs.as_ptr(), caps.as_ptr(), nouts.as_mut_ptr(),
                                    infos.as_mut_ptr(), statuses.as_mut_ptr(),
                                    if devices.is_empty() { std::ptr::null() } else { devices.as_ptr() }, devices.len() as i32,
                                    streams_per_device)
    };
    // nothing decoded at all (argument and settings errors come back before any status is written): an error
    if st != 0 && statuses.iter().all(|&v| v == st || v == -1) { return Err(to_error(st)); }
    Ok(outs.into_iter().enumerate().map(|(i, mut o)| {
        if statuses[i] != 0 { return Err(to_error(statuses[i])); }
        o.truncate(nouts[i] as usize);
        Ok((o, infos[i].low, infos[i].high))
    }).collect())
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
