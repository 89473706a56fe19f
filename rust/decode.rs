//! Replacement body for `src/decode.rs::decode` (decode.rs:43-162) of martinber/noaa-apt: same signature,
//! the work is done by libaptb200 on an H100.  SOURCE ONLY (never compiled here: no Rust toolchain in the
//! image).  `find_sync`, `generate_sync_frame` and the constants of decode.rs stay as they are.

use std::ffi::CStr;
use std::os::raw::{c_char, c_float, c_void};

use crate::aptb200_sys as sys;
use crate::config;
use crate::context::Context;
use crate::dsp::{Rate, Signal};
use crate::err;

/// apt_status -> err::Error (err.rs:9-44): 1-4 and 10 are `Internal`, 5 is `RateOverflow`.
pub(crate) fn to_error(status: i32) -> err::Error {
    let msg = unsafe {
        let p = sys::apt_last_error();
        let s = if p.is_null() { String::new() } else { CStr::from_ptr(p).to_string_lossy().into_owned() };
        if s.is_empty() { CStr::from_ptr(sys::apt_strerror(status)).to_string_lossy().into_owned() } else { s }
    };
    match status {
        sys::APT_ERR_RATE_OVERFLOW => err::Error::RateOverflow(msg),
        sys::APT_ERR_BAD_ARG | sys::APT_ERR_CAPACITY => err::Error::InvalidInput(msg),
        _ => err::Error::Internal(msg),
    }
}

/// Context::status is `FnMut + 'static`, not `Send` (context.rs:122): the library fires the callback on the
/// calling thread, at the reference's five points (decode.rs:63,87,93,107/136,154).
unsafe extern "C" fn status_trampoline(progress: c_float, description: *const c_char, user: *mut c_void) {
    let context = &mut *(user as *mut Context);
    let text = if description.is_null() { String::new() } else { CStr::from_ptr(description).to_string_lossy().into_owned() };
    context.status(progress, text);
}

pub fn decode(
    context: &mut Context,
    settings: &config::Settings,
    signal: &Signal,
    input_rate: Rate,
    sync: bool,
) -> err::Result<Signal> {
    let s = sys::apt_settings {
        work_rate: settings.work_rate,
        resample_atten: settings.resample_atten,
        resample_delta_freq: settings.resample_delta_freq,
        resample_cutout: settings.resample_cutout,
        demodulation_atten: settings.demodulation_atten,
    };
    let mut bound: u64 = 0;
    let st = unsafe { sys::apt_decode_len_bound(signal.len() as u64, input_rate.get_hz(), &s, &mut bound) };
    if st != sys::APT_OK {
        return Err(to_error(st));
    }
    let mut out: Signal = vec![0_f32; bound.max(1) as usize];
    let mut n: u64 = 0;
    let st = unsafe {
        sys::apt_decode(
            signal.as_ptr(), signal.len() as u64, input_rate.get_hz(), &s, sync as i32,
            out.as_mut_ptr(), out.len() as u64, &mut n,
            Some(status_trampoline), context as *mut Context as *mut c_void,
        )
    };
    if st != sys::APT_OK {
        return Err(to_error(st));
    }
    out.truncate(n as usize);
    Ok(out)
}

/// `decode` with tracked sync (DESIGN.md "Tracked sync", `apt_decoder_set_sync_mode`): the row period followed through
/// the whole pass instead of the reference's per-row maximum.  `track` = (delta, lambda); `None` takes the defaults
/// (2, 0.25).  Runs on a decoder of its own on device 0.
pub fn decode_tracked(
    settings: &config::Settings,
    signal: &Signal,
    input_rate: Rate,
    track: Option<(u32, f32)>,
) -> err::Result<Signal> {
    let s = sys::apt_settings {
        work_rate: settings.work_rate,
        resample_atten: settings.resample_atten,
        resample_delta_freq: settings.resample_delta_freq,
        resample_cutout: settings.resample_cutout,
        demodulation_atten: settings.demodulation_atten,
    };
    let mut ts = sys::apt_track_settings { delta: 0, lambda: 0.0 };
    unsafe { sys::apt_default_track_settings(&mut ts) };
    if let Some((delta, lambda)) = track {
        ts = sys::apt_track_settings { delta, lambda };
    }
    let mut bound: u64 = 0;
    let st = unsafe { sys::apt_decode_len_bound(signal.len() as u64, input_rate.get_hz(), &s, &mut bound) };
    if st != sys::APT_OK {
        return Err(to_error(st));
    }
    let mut dec: *mut sys::apt_decoder = std::ptr::null_mut();
    let st = unsafe { sys::apt_decoder_create(0, input_rate.get_hz(), &s, signal.len() as u64, &mut dec) };
    if st != sys::APT_OK {
        return Err(to_error(st));
    }
    let mut out: Signal = vec![0_f32; bound.max(1) as usize];
    let mut n: u64 = 0;
    let st = unsafe {
        let mut st = sys::apt_decoder_set_sync_mode(dec, sys::APT_SYNC_TRACK, &ts);
        if st == sys::APT_OK {
            st = sys::apt_decoder_submit_host(dec, signal.as_ptr() as *const c_void, sys::APT_F32, signal.len() as u64, 1,
                                              out.as_mut_ptr(), out.len() as u64);
        }
        if st == sys::APT_OK {
            st = sys::apt_decoder_wait(dec, &mut n);
        }
        sys::apt_decoder_destroy(dec);
        st
    };
    if st != sys::APT_OK {
        return Err(to_error(st));
    }
    out.truncate(n as usize);
    Ok(out)
}
