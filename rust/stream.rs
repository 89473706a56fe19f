//! Live decoding for noaa-apt: `Stream` wraps libaptb200's apt_stream (push audio as it arrives, get the image rows
//! that became final).  The rows of all pushes plus `finish` equal `decode::decode` on the whole recording, bit for bit.
//! SOURCE ONLY (never compiled here: no Rust toolchain in the image).  INTEGRATION.md shows a TCP/UDP audio loop on it.

use std::os::raw::c_void;
use std::ptr;

use crate::aptb200_sys as sys;
use crate::config;
use crate::decode::to_error;
use crate::dsp::{Rate, Signal};
use crate::err;

pub struct Stream {
    st: *mut sys::apt_stream,
    image: Option<(u64, i32)>,                 // image output: (max_rows, bytes per pixel)
    png: Option<sys::apt_png_settings>,        // PNG output
}

/// What `finish_image` returns: the rows `finish` would return, the image (rows * 2080 pixels of 1 grey or 4 RGBA bytes,
/// or the PNG file) and the contrast info.
pub struct PassImage {
    pub rows: Signal,
    pub image: Vec<u8>,
    pub info: sys::apt_image_info,
}

// The stream is used from one thread at a time; moving it to another thread is fine.
unsafe impl Send for Stream {}

impl Stream {
    /// `max_push`: samples one internal step takes (larger pushes are split); the device memory depends on it.
    pub fn new(input_rate: Rate, settings: &config::Settings, sync: bool, max_push: u64, device: i32) -> err::Result<Stream> {
        let s = sys::apt_settings {
            work_rate: settings.work_rate,
            resample_atten: settings.resample_atten,
            resample_delta_freq: settings.resample_delta_freq,
            resample_cutout: settings.resample_cutout,
            demodulation_atten: settings.demodulation_atten,
        };
        let mut st: *mut sys::apt_stream = ptr::null_mut();
        let rc = unsafe { sys::apt_stream_create(device, input_rate.get_hz(), &s, sync as i32, max_push, &mut st) };
        if rc != sys::APT_OK {
            return Err(to_error(rc));
        }
        Ok(Stream { st, image: None, png: None })
    }

    fn rows(&mut self, n: u64, call: impl FnOnce(*mut f32, u64, *mut u64) -> i32) -> err::Result<Signal> {
        let mut cap: u64 = 0;
        let rc = unsafe { sys::apt_stream_push_bound(self.st, n, &mut cap) };
        if rc != sys::APT_OK {
            return Err(to_error(rc));
        }
        let mut out: Signal = vec![0_f32; cap.max(1) as usize];
        let mut got: u64 = 0;
        let rc = call(out.as_mut_ptr(), out.len() as u64, &mut got);
        if rc != sys::APT_OK {
            return Err(to_error(rc));
        }
        out.truncate(got as usize);
        Ok(out)
    }

    /// f32 samples (a `Signal`) -> the rows (2080 pixels each, concatenated) that became final.
    pub fn push(&mut self, samples: &[f32]) -> err::Result<Signal> {
        let st = self.st;
        self.rows(samples.len() as u64, |o, c, k| unsafe {
            sys::apt_stream_push(st, samples.as_ptr() as *const c_void, sys::APT_F32, samples.len() as u64, o, c, k)
        })
    }

    /// PCM16 samples as a WAV or a sound card delivers them.
    pub fn push_pcm16(&mut self, samples: &[i16]) -> err::Result<Signal> {
        let st = self.st;
        self.rows(samples.len() as u64, |o, c, k| unsafe {
            sys::apt_stream_push(st, samples.as_ptr() as *const c_void, sys::APT_PCM16, samples.len() as u64, o, c, k)
        })
    }

    /// A stream fed with I/Q (apt_stream_create_iq): push_iq() only; max_push counts I/Q samples.
    pub fn new_iq(iq: &sys::apt_iq_settings, settings: &config::Settings, sync: bool, max_push: u64, device: i32)
                  -> err::Result<Stream> {
        let s = sys::apt_settings {
            work_rate: settings.work_rate,
            resample_atten: settings.resample_atten,
            resample_delta_freq: settings.resample_delta_freq,
            resample_cutout: settings.resample_cutout,
            demodulation_atten: settings.demodulation_atten,
        };
        let mut st: *mut sys::apt_stream = ptr::null_mut();
        let rc = unsafe { sys::apt_stream_create_iq(device, iq, &s, sync as i32, max_push, &mut st) };
        if rc != sys::APT_OK {
            return Err(to_error(rc));
        }
        Ok(Stream { st, image: None, png: None })
    }

    /// I/Q samples of an I/Q stream (cu8 / cs16 / cf32 pushes may be mixed).
    pub fn push_iq(&mut self, samples: &crate::iq::Iq) -> err::Result<Signal> {
        let st = self.st;
        let (p, fmt, n) = samples.raw();
        self.rows(n, |o, c, k| unsafe { sys::apt_stream_push(st, p, fmt, n, o, c, k) })
    }

    /// The remaining rows; the error `decode` would return (too short, too few sync frames) means the rows returned
    /// so far are not an image and are discarded.
    pub fn finish(&mut self) -> err::Result<Signal> {
        let st = self.st;
        self.rows(0, |o, c, k| unsafe { sys::apt_stream_finish(st, o, c, k) })
    }

    /// Starts a new recording with the same plan and device memory.
    pub fn reset(&mut self) -> err::Result<()> {
        let rc = unsafe { sys::apt_stream_reset(self.st) };
        if rc != sys::APT_OK { Err(to_error(rc)) } else { Ok(()) }
    }

    /// Sync positions decided so far (after `finish`: those of `decode::find_sync`).
    pub fn positions(&self) -> err::Result<Vec<u64>> {
        let mut n: usize = 0;
        let rc = unsafe { sys::apt_stream_sync_positions(self.st, ptr::null_mut(), 0, &mut n) };
        if rc != sys::APT_OK {
            return Err(to_error(rc));
        }
        let mut pos = vec![0_u64; n];
        let rc = unsafe { sys::apt_stream_sync_positions(self.st, pos.as_mut_ptr(), pos.len(), &mut n) };
        if rc != sys::APT_OK {
            return Err(to_error(rc));
        }
        Ok(pos)
    }

    /// Image output, before the first push of a pass: `finish_image` also returns the image of `process` (`ps`) for a pass
    /// of up to `max_rows` rows.  `None` switches image and PNG output off and frees their device memory.
    pub fn set_process_mode(&mut self, ps: Option<&sys::apt_process_settings>, max_rows: u64) -> err::Result<()> {
        let p = ps.map_or(ptr::null(), |p| p as *const _);
        let rc = unsafe { sys::apt_stream_set_process_mode(self.st, p, max_rows) };
        if rc != sys::APT_OK {
            return Err(to_error(rc));
        }
        self.image = ps.map(|p| (max_rows, if p.rgba != 0 { 4 } else { 1 }));
        self.png = None;
        Ok(())
    }

    /// PNG output (needs process mode): `finish_image` returns the PNG file's bytes, ready to write.
    pub fn set_png_mode(&mut self, png: Option<&sys::apt_png_settings>) -> err::Result<()> {
        let p = png.map_or(ptr::null(), |p| p as *const _);
        let rc = unsafe { sys::apt_stream_set_png_mode(self.st, p) };
        if rc != sys::APT_OK {
            return Err(to_error(rc));
        }
        self.png = png.copied();
        Ok(())
    }

    /// `finish` plus the image of the pass (equal to `decode_image` / `decode_to_png` on the whole recording).
    pub fn finish_image(&mut self) -> err::Result<PassImage> {
        let (max_rows, bpp) = self.image.unwrap_or((0, 1));
        let mut cap: u64 = max_rows * 2080 * bpp as u64;
        if let Some(png) = self.png {
            let rc = unsafe { sys::apt_png_bound(2080, max_rows.max(1) as u32, bpp, &png, &mut cap) };
            if rc != sys::APT_OK {
                return Err(to_error(rc));
            }
        }
        let mut image = vec![0_u8; cap.max(1) as usize];
        let mut info = sys::apt_image_info::default();
        let mut n: u64 = 0;
        let st = self.st;
        let rows = self.rows(0, |o, c, k| unsafe {
            sys::apt_stream_finish_image(st, o, c, k, image.as_mut_ptr(), image.len() as u64, &mut n, &mut info)
        })?;
        image.truncate(n as usize);
        Ok(PassImage { rows, image, info })
    }

    pub fn info(&self) -> err::Result<sys::apt_stream_info> {
        let mut i = sys::apt_stream_info::default();
        let rc = unsafe { sys::apt_stream_get_info(self.st, &mut i) };
        if rc != sys::APT_OK { Err(to_error(rc)) } else { Ok(i) }
    }
}

impl Drop for Stream {
    fn drop(&mut self) {
        unsafe { sys::apt_stream_destroy(self.st) }
    }
}
