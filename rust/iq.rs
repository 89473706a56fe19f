//! Decoding straight from SDR I/Q for noaa-apt (DESIGN.md §10): FM demodulation on the device, then decode, or a live
//! `Stream` fed with I/Q from an RTL-SDR.  SOURCE ONLY (never compiled here: no Rust toolchain in the image).

use std::ptr;

use crate::aptb200_sys as sys;
use crate::config;
use crate::decode::to_error;
use crate::dsp::Signal;
use crate::err;

/// The I/Q sample formats, interleaved I, Q.
pub enum Iq<'a> {
    Cu8(&'a [u8]),     // rtl_sdr / librtlsdr
    Cs16(&'a [i16]),   // SDR# / SDR++ baseband WAV
    Cf32(&'a [f32]),   // GQRX, GNU Radio file sink
}

impl<'a> Iq<'a> {
    pub(crate) fn raw(&self) -> (*const std::os::raw::c_void, i32, u64) {
        match self {
            Iq::Cu8(x) => (x.as_ptr() as *const _, sys::APT_CU8, (x.len() / 2) as u64),
            Iq::Cs16(x) => (x.as_ptr() as *const _, sys::APT_CS16, (x.len() / 2) as u64),
            Iq::Cf32(x) => (x.as_ptr() as *const _, sys::APT_CF32, (x.len() / 2) as u64),
        }
    }
}

fn check(rc: i32) -> err::Result<()> {
    if rc == sys::APT_OK { Ok(()) } else { Err(to_error(rc)) }
}

/// apt_iq_default_settings: channel filter 22 kHz / 8 kHz / 40 dB, audio rate the smallest iq_rate / D >= 48 kHz.
pub fn default_settings(iq_rate: u32, offset_hz: i32) -> err::Result<sys::apt_iq_settings> {
    let mut s = sys::apt_iq_settings::default();
    check(unsafe { sys::apt_iq_default_settings(iq_rate, offset_hz, &mut s) })?;
    Ok(s)
}

/// The I/Q stage alone: instantaneous frequency in Hz at s.audio_rate.
pub fn fm_demod(iq: &Iq, s: &sys::apt_iq_settings) -> err::Result<Signal> {
    let (p, fmt, n) = iq.raw();
    let mut len: u64 = 0;
    check(unsafe { sys::apt_fm_demod_len(n, s, &mut len) })?;
    let mut out = vec![0f32; len.max(1) as usize];
    let mut got: u64 = 0;
    check(unsafe { sys::apt_fm_demod(p, fmt, n, s, out.as_mut_ptr(), out.len() as u64, &mut got) })?;
    out.truncate(got as usize);
    Ok(out)
}

/// decode::decode of the demodulated I/Q at s.audio_rate; the audio stays on the GPU.
pub fn decode_iq(iq: &Iq, s: &sys::apt_iq_settings, settings: &config::Settings, sync: bool) -> err::Result<Signal> {
    let (p, fmt, n) = iq.raw();
    let st = sys::apt_settings {
        work_rate: settings.work_rate,
        resample_atten: settings.resample_atten,
        resample_delta_freq: settings.resample_delta_freq,
        resample_cutout: settings.resample_cutout,
        demodulation_atten: settings.demodulation_atten,
    };
    let (mut len, mut bound, mut got) = (0u64, 0u64, 0u64);
    check(unsafe { sys::apt_fm_demod_len(n, s, &mut len) })?;
    check(unsafe { sys::apt_decode_len_bound(len, s.audio_rate, &st, &mut bound) })?;
    let mut out = vec![0f32; bound.max(1) as usize];
    check(unsafe {
        sys::apt_decode_iq(p, fmt, n, s, &st, sync as i32, out.as_mut_ptr(), out.len() as u64, &mut got, None, ptr::null_mut())
    })?;
    out.truncate(got as usize);
    Ok(out)
}
