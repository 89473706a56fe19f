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

/// What a `Watch` hands its closure: an AOS, a SEGMENT, or at LOS the pass's decode (`data`: the PNG file, or the f32
/// rows as bytes without image output; `Err` the pass's own failure, e.g. more rows than `max_rows`).
pub enum WatchEvent<'a> {
    Aos { index: u32, pass: sys::apt_pass },
    Los { index: u32, pass: sys::apt_pass, rows: u64, data: err::Result<&'a [u8]>, info: sys::apt_image_info },
    Segment { start: u64 },
}

struct Handler<'f> {
    f: Box<dyn FnMut(WatchEvent) + 'f>,
}

unsafe fn watch_event<'a>(e: &'a sys::apt_watch_event) -> WatchEvent<'a> {
    match e.ev.kind {
        sys::APT_PASS_AOS => WatchEvent::Aos { index: e.index, pass: e.ev.pass },
        sys::APT_PASS_SEGMENT => WatchEvent::Segment { start: e.ev.pass.start },
        _ => WatchEvent::Los {
            index: e.index,
            pass: e.ev.pass,
            rows: e.rows,
            data: if e.status == sys::APT_OK {
                Ok(std::slice::from_raw_parts(e.data as *const u8, e.bytes as usize))
            } else {
                Err(to_error(e.status))
            },
            info: e.info,
        },
    }
}

unsafe extern "C" fn watch_trampoline(ev: *const sys::apt_watch_event, user: *mut c_void) {
    let h = &mut *(user as *mut Handler);
    let out = watch_event(&*ev);
    // a panic must not unwind into the library
    let _ = std::panic::catch_unwind(std::panic::AssertUnwindSafe(|| (h.f)(out)));
}

/// A continuous feed (16-bit samples as they arrive) watched for satellite passes, each ended in its PNG file (`png`)
/// or its f32 rows, in fixed device memory (DESIGN.md §13).  The closure runs on the pushing thread.
pub struct Watch<'f> {
    h: *mut sys::apt_watch,
    handler: Box<Handler<'f>>,
}

impl<'f> Watch<'f> {
    pub fn new(input_rate: Rate, settings: &config::Settings, search: &sys::apt_pass_search,
               image: Option<(&sys::apt_process_settings, Option<&sys::apt_png_settings>)>, max_rows: u64, device: i32,
               on_event: impl FnMut(WatchEvent) + 'f) -> err::Result<Watch<'f>> {
        let s = sys::apt_settings::from(settings);
        let ws = sys::apt_watch_settings {
            sync: 1,
            search: *search,
            ps: image.map_or(ptr::null(), |(ps, _)| ps as *const _),
            png: image.and_then(|(_, png)| png).map_or(ptr::null(), |p| p as *const _),
            max_rows,
            max_push: 0,
        };
        let mut handler = Box::new(Handler { f: Box::new(on_event) });
        let mut h = ptr::null_mut();
        check(unsafe { sys::apt_watch_create(device, input_rate.get_hz(), &s, &ws, Some(watch_trampoline),
                                             &mut *handler as *mut Handler as *mut c_void, &mut h) })?;
        Ok(Watch { h, handler })
    }

    /// The new windows' quality; events reach the closure during the call.
    pub fn push(&mut self, pcm: &[i16]) -> err::Result<Vec<f32>> {
        let mut cap = 0u64;
        check(unsafe { sys::apt_watch_push_bound(self.h, pcm.len() as u64, &mut cap) })?;
        let mut q = vec![0f32; cap.max(1) as usize];
        let mut nq = 0u64;
        check(unsafe { sys::apt_watch_push(self.h, pcm.as_ptr() as *const c_void, sys::APT_PCM16, pcm.len() as u64,
                                           q.as_mut_ptr(), q.len() as u64, &mut nq) })?;
        q.truncate(nq as usize);
        Ok(q)
    }

    /// The end of the feed: the tail windows and the LOS of a pass still open.
    pub fn finish(&mut self) -> err::Result<Vec<f32>> {
        let mut cap = 0u64;
        check(unsafe { sys::apt_watch_push_bound(self.h, 0, &mut cap) })?;
        let mut q = vec![0f32; cap.max(1) as usize];
        let mut nq = 0u64;
        check(unsafe { sys::apt_watch_finish(self.h, q.as_mut_ptr(), q.len() as u64, &mut nq) })?;
        q.truncate(nq as usize);
        Ok(q)
    }

    pub fn reset(&mut self) -> err::Result<()> { check(unsafe { sys::apt_watch_reset(self.h) }) }

    pub fn info(&self) -> err::Result<sys::apt_watch_info> {
        let mut i = sys::apt_watch_info::default();
        check(unsafe { sys::apt_watch_get_info(self.h, &mut i) })?;
        Ok(i)
    }
}

impl<'f> Drop for Watch<'f> {
    fn drop(&mut self) {
        unsafe { sys::apt_watch_destroy(self.h) };
        let _ = &self.handler;   // freed after the watcher, which holds its address
    }
}

/// One SDR's I/Q feed (cu8 as rtl_sdr writes it) watched for passes on up to 8 channels at once (DESIGN.md §14): channel
/// c behaves as a `Watch` on the FM audio at `offsets[c]` Hz from the tuned centre.  The closure gets the channel and the
/// event; event positions are audio samples of the channel.
pub struct IqWatch<'f> {
    h: *mut sys::apt_watch_iq,
    count: usize,
    handler: Box<IqHandler<'f>>,
}

struct IqHandler<'f> {
    f: Box<dyn FnMut(usize, WatchEvent) + 'f>,
}

unsafe extern "C" fn watch_iq_trampoline(channel: i32, ev: *const sys::apt_watch_event, user: *mut c_void) {
    let h = &mut *(user as *mut IqHandler);
    let out = watch_event(&*ev);
    let _ = std::panic::catch_unwind(std::panic::AssertUnwindSafe(|| (h.f)(channel as usize, out)));
}

impl<'f> IqWatch<'f> {
    pub fn new(iq: &sys::apt_iq_settings, offsets: &[i32], settings: &config::Settings, search: &sys::apt_pass_search,
               image: Option<(&sys::apt_process_settings, Option<&sys::apt_png_settings>)>, max_rows: u64, device: i32,
               on_event: impl FnMut(usize, WatchEvent) + 'f) -> err::Result<IqWatch<'f>> {
        let s = sys::apt_settings::from(settings);
        let ws = sys::apt_watch_settings {
            sync: 1,
            search: *search,
            ps: image.map_or(ptr::null(), |(ps, _)| ps as *const _),
            png: image.and_then(|(_, png)| png).map_or(ptr::null(), |p| p as *const _),
            max_rows,
            max_push: 0,
        };
        let mut handler = Box::new(IqHandler { f: Box::new(on_event) });
        let mut h = ptr::null_mut();
        check(unsafe { sys::apt_watch_iq_create(device, iq, offsets.as_ptr(), offsets.len() as i32, &s, &ws,
                                                Some(watch_iq_trampoline),
                                                &mut *handler as *mut IqHandler as *mut c_void, &mut h) })?;
        Ok(IqWatch { h, count: offsets.len(), handler })
    }

    fn split(&self, q: Vec<f32>, cap: usize, nq: &[u64]) -> Vec<Vec<f32>> {
        (0..self.count).map(|c| q[c * cap..c * cap + nq[c] as usize].to_vec()).collect()
    }

    /// Interleaved cu8 I/Q: each channel's new windows' quality; events reach the closure during the call.
    pub fn push(&mut self, cu8: &[u8]) -> err::Result<Vec<Vec<f32>>> {
        let n = (cu8.len() / 2) as u64;
        let mut cap = 0u64;
        check(unsafe { sys::apt_watch_iq_push_bound(self.h, n, &mut cap) })?;
        let cap = cap.max(1) as usize;
        let mut q = vec![0f32; cap * self.count];
        let mut nq = vec![0u64; self.count];
        check(unsafe { sys::apt_watch_iq_push(self.h, cu8.as_ptr() as *const c_void, sys::APT_CU8, n, q.as_mut_ptr(),
                                              cap as u64, nq.as_mut_ptr()) })?;
        Ok(self.split(q, cap, &nq))
    }

    /// The end of the feed on every channel.
    pub fn finish(&mut self) -> err::Result<Vec<Vec<f32>>> {
        let mut cap = 0u64;
        check(unsafe { sys::apt_watch_iq_push_bound(self.h, 0, &mut cap) })?;
        let cap = cap.max(1) as usize;
        let mut q = vec![0f32; cap * self.count];
        let mut nq = vec![0u64; self.count];
        check(unsafe { sys::apt_watch_iq_finish(self.h, q.as_mut_ptr(), cap as u64, nq.as_mut_ptr()) })?;
        Ok(self.split(q, cap, &nq))
    }

    pub fn reset(&mut self) -> err::Result<()> { check(unsafe { sys::apt_watch_iq_reset(self.h) }) }

    pub fn info(&self, channel: usize) -> err::Result<sys::apt_watch_info> {
        let mut i = sys::apt_watch_info::default();
        check(unsafe { sys::apt_watch_iq_get_info(self.h, channel as i32, &mut i) })?;
        Ok(i)
    }
}

impl<'f> Drop for IqWatch<'f> {
    fn drop(&mut self) {
        unsafe { sys::apt_watch_iq_destroy(self.h) };
        let _ = &self.handler;   // freed after the watcher, which holds its address
    }
}
