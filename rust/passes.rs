//! Finding the satellite passes in a long recording and decoding each one from a single upload (DESIGN.md §12): what a
//! station recording all day or overnight needs before noaa-apt's per-pass decode.  SOURCE ONLY (never compiled here: no
//! Rust toolchain in the image).

use std::os::raw::c_void;
use std::ptr;

use crate::aptb200_sys as sys;
use crate::config;
use crate::decode::to_error;
use crate::dsp::Rate;
use crate::err;
use crate::noaa_apt::{ColorSettings, Contrast, Rotate};

fn check(rc: i32) -> err::Result<()> {
    if rc == sys::APT_OK { Ok(()) } else { Err(to_error(rc)) }
}

/// The pass rule on a quality array (host only).  Zero fields of `search` take the defaults (enter 0.30, exit 0.15,
/// max_gap 30 s, min_length 60 s).
pub fn find_passes_quality(q: &[f32], n: u64, input_rate: Rate, search: &sys::apt_pass_search) -> err::Result<Vec<sys::apt_pass>> {
    let mut count = 0u32;
    let rc = unsafe { sys::apt_find_passes_quality(q.as_ptr(), q.len() as u64, n, input_rate.get_hz(), search, ptr::null_mut(), 0,
                                                   &mut count) };
    if rc != sys::APT_ERR_CAPACITY { check(rc)?; }
    let mut out = vec![sys::apt_pass::default(); count as usize];
    if count > 0 {
        check(unsafe { sys::apt_find_passes_quality(q.as_ptr(), q.len() as u64, n, input_rate.get_hz(), search, out.as_mut_ptr(),
                                                    count, &mut count) })?;
    }
    Ok(out)
}

/// A recording (16-bit samples of the WAV) kept in device memory from `new` until it is dropped.
pub struct Recording {
    h: *mut sys::apt_recording,
    n: u64,
    rate: Rate,
    settings: sys::apt_settings,
}

impl Recording {
    pub fn new(pcm: &[i16], input_rate: Rate, settings: &config::Settings, device: i32) -> err::Result<Recording> {
        let s = sys::apt_settings::from(settings);
        let mut h = ptr::null_mut();
        check(unsafe { sys::apt_recording_create(device, pcm.as_ptr() as *const c_void, sys::APT_PCM16, pcm.len() as u64,
                                                 input_rate.get_hz(), &s, &mut h) })?;
        Ok(Recording { h, n: pcm.len() as u64, rate: input_rate, settings: s })
    }

    pub fn info(&self) -> err::Result<sys::apt_recording_info> {
        let mut i = sys::apt_recording_info::default();
        check(unsafe { sys::apt_recording_get_info(self.h, &mut i) })?;
        Ok(i)
    }

    /// q: the correlation of each image row of the envelope with the next one.
    pub fn quality(&self) -> err::Result<Vec<f32>> {
        let mut nq = 0u64;
        check(unsafe { sys::apt_recording_quality(self.h, ptr::null_mut(), 0, &mut nq) })?;
        let mut q = vec![0f32; nq as usize];
        if nq > 0 { check(unsafe { sys::apt_recording_quality(self.h, q.as_mut_ptr(), nq, &mut nq) })?; }
        Ok(q)
    }

    pub fn find_passes(&self, search: &sys::apt_pass_search) -> err::Result<Vec<sys::apt_pass>> {
        find_passes_quality(&self.quality()?, self.n, self.rate, search)
    }

    /// The PNG file of each range, as `image::decode_to_png` of that slice gives it: Ok(bytes) or the range's own error.
    pub fn decode_png(&self, ranges: &[sys::apt_pass], sync: bool, contrast: &Contrast, rotate: &Rotate,
                      color: Option<&ColorSettings>) -> err::Result<Vec<err::Result<Vec<u8>>>> {
        let (mode, percent, rotate, palette, tune) = crate::image::png_process_parts(contrast, rotate, color)?;
        let ps = sys::apt_process_settings { contrast: mode, percent, rotate,
                                             palette: palette.as_ref().map_or(ptr::null(), |p| p.as_ptr()), tune, rgba: 1 };
        let png = sys::apt_png_settings::default();
        let k = ranges.len();
        let mut bufs = Vec::with_capacity(k);
        for r in ranges {
            let mut bound = 0u64;
            check(unsafe { sys::apt_decode_len_bound(r.end.saturating_sub(r.start), self.rate.get_hz(), &self.settings, &mut bound) })?;
            let rows = (bound / crate::decode::PX_PER_ROW as u64).max(1);
            let mut cap = 0u64;
            check(unsafe { sys::apt_png_bound(crate::decode::PX_PER_ROW as u32, rows as u32, 4, &png, &mut cap) })?;
            bufs.push(vec![0u8; cap.max(1) as usize]);
        }
        let outs: Vec<*mut c_void> = bufs.iter_mut().map(|b| b.as_mut_ptr() as *mut c_void).collect();
        let caps: Vec<u64> = bufs.iter().map(|b| b.len() as u64).collect();
        let mut nouts = vec![0u64; k];
        let mut statuses = vec![0i32; k];
        let rc = unsafe { sys::apt_recording_decode(self.h, ranges.as_ptr(), k as u32, sync as i32, &ps, &png, outs.as_ptr(),
                                                    caps.as_ptr(), nouts.as_mut_ptr(), ptr::null_mut(), statuses.as_mut_ptr()) };
        if rc == sys::APT_ERR_BAD_ARG && statuses.iter().all(|&s| s == rc) { return Err(to_error(rc)); }
        Ok(bufs.into_iter().zip(nouts).zip(statuses).map(|((mut b, n), st)| {
            if st == sys::APT_OK { b.truncate(n as usize); Ok(b) } else { Err(to_error(st)) }
        }).collect())
    }
}

impl Drop for Recording {
    fn drop(&mut self) { unsafe { sys::apt_recording_destroy(self.h) } }
}
