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

/// The averaged power spectrum (fftshifted, bin b at (b - nfft/2) iq_rate / nfft Hz) and the number of segments used.
pub fn spectrum(iq: &Iq, iq_rate: u32, nfft: u32, max_segments: u32) -> err::Result<(Vec<f32>, u32)> {
    let (p, fmt, n) = iq.raw();
    let ss = sys::apt_spectrum_settings { nfft, max_segments };
    let mut psd = vec![0f32; nfft as usize];
    let mut nseg: u32 = 0;
    check(unsafe { sys::apt_iq_spectrum(p, fmt, n, iq_rate, &ss, psd.as_mut_ptr(), psd.len() as u64, &mut nseg) })?;
    Ok((psd, nseg))
}

/// The carriers of a recording by descending SNR; `offset_hz` of each is ready for `apt_iq_settings`.
pub fn find_carriers(iq: &Iq, s: &sys::apt_iq_settings, cs: &sys::apt_carrier_search) -> err::Result<Vec<sys::apt_carrier>> {
    let (p, fmt, n) = iq.raw();
    let mut out = vec![sys::apt_carrier::default(); (s.iq_rate / 40_000 + 2) as usize];   // carriers are > 40 kHz apart
    let mut count: u32 = 0;
    check(unsafe { sys::apt_iq_find_carriers(p, fmt, n, s, cs, out.as_mut_ptr(), out.len() as u32, &mut count) })?;
    out.truncate(count as usize);
    Ok(out)
}

/// Every APT carrier of a recording decoded from one upload: (carrier, its rows or the error of its decode).
pub fn decode_iq_auto(iq: &Iq, s: &sys::apt_iq_settings, cs: &sys::apt_carrier_search, settings: &config::Settings,
                      sync: bool, max_channels: usize) -> err::Result<Vec<(sys::apt_carrier, err::Result<Signal>)>> {
    let (p, fmt, n) = iq.raw();
    let st = sys::apt_settings {
        work_rate: settings.work_rate,
        resample_atten: settings.resample_atten,
        resample_delta_freq: settings.resample_delta_freq,
        resample_cutout: settings.resample_cutout,
        demodulation_atten: settings.demodulation_atten,
    };
    let s0 = sys::apt_iq_settings { offset_hz: 0, ..*s };
    let (mut len, mut bound) = (0u64, 0u64);
    check(unsafe { sys::apt_fm_demod_len(n, &s0, &mut len) })?;
    check(unsafe { sys::apt_decode_len_bound(len, s.audio_rate, &st, &mut bound) })?;
    let k = max_channels.max(1);
    let mut bufs: Vec<Vec<f32>> = (0..k).map(|_| vec![0f32; bound.max(1) as usize]).collect();
    let outs: Vec<*mut f32> = bufs.iter_mut().map(|b| b.as_mut_ptr()).collect();
    let caps = vec![bound.max(1); k];
    let mut nouts = vec![0u64; k];
    let mut statuses = vec![0i32; k];
    let mut found = vec![sys::apt_carrier::default(); k];
    let mut nfound: u32 = 0;
    let rc = unsafe {
        sys::apt_decode_iq_auto(p, fmt, n, s, cs, &st, sync as i32, found.as_mut_ptr(), k as u32, &mut nfound, outs.as_ptr(),
                                caps.as_ptr(), nouts.as_mut_ptr(), statuses.as_mut_ptr())
    };
    // an error before any channel was decoded (bad arguments, too short) is the call's; otherwise each channel has its own
    if rc != sys::APT_OK && (nfound == 0 || statuses[..nfound as usize].iter().all(|&x| x == rc)) {
        return Err(to_error(rc));
    }
    Ok(found.into_iter().zip(bufs).zip(nouts.iter().zip(statuses.iter())).take(nfound as usize)
        .map(|((c, mut b), (&got, &status))| {
            (c, if status == sys::APT_OK { b.truncate(got as usize); Ok(b) } else { Err(to_error(status)) })
        })
        .collect())
}
