"""First-stage geometry without a GPU: apt_stream_geometry and apt_decode_len_bound for one input rate per first-stage
kind (front.hpp), plus the fast and slow profiles, pinned to the values they have always had.

Kinds chosen by the standard profile: 48 000 Hz tiled, 192 000 Hz uniform-tap, 11 025 Hz phase-major, 8000 Hz generic,
24 960 Hz decimate (L = 1); 11 025 Hz in the fast and slow profiles runs on the generic kernel, 48 000 Hz on the tiled one.
The stream's device bytes include the first stage's tables and its input and envelope windows, whose sizes follow from
the kind's unit geometry; a change to a plan or a unit shows up here.
"""
import pytest

import noaa_apt_b200 as na

# (rate, profile): decode_len_bound for n = 20 s of samples + 7 and for n = 9 067 017
BOUNDS = {
    (48000, 'standard'): [81120, 784160],
    (192000, 'standard'): [81120, 195520],
    (11025, 'standard'): [81120, 3419520],
    (8000, 'standard'): [83200, 4713280],
    (24960, 'standard'): [83200, 1510080],
    (11025, 'fast'): [83200, 3419520],
    (11025, 'slow'): [81120, 3419520],
    (48000, 'fast'): [81120, 784160],
    (48000, 'slow'): [81120, 784160],
}

# (rate, profile, sync, max_push, latency_work, device_bytes)
GEOMETRY = [
    (48000, 'standard', True, 4800, 4993, 719780),
    (48000, 'standard', True, 48000, 4993, 1303212),
    (48000, 'standard', False, 4800, 0, 515708),
    (48000, 'standard', False, 48000, 0, 1009284),
    (192000, 'standard', True, 4800, 4993, 414168),
    (192000, 'standard', True, 48000, 4993, 879864),
    (192000, 'standard', False, 4800, 0, 310896),
    (192000, 'standard', False, 48000, 0, 754128),
    (11025, 'standard', True, 4800, 4993, 2293040),
    (11025, 'standard', True, 48000, 4993, 3370120),
    (11025, 'standard', False, 4800, 0, 1303032),
    (11025, 'standard', False, 48000, 0, 1988904),
    (8000, 'standard', True, 4800, 4993, 371512),
    (8000, 'standard', True, 48000, 4993, 1703780),
    (8000, 'standard', False, 4800, 0, 223592),
    (8000, 'standard', False, 48000, 0, 1016724),
    (24960, 'standard', True, 4800, 4993, 402124),
    (24960, 'standard', True, 48000, 4993, 1204696),
    (24960, 'standard', False, 4800, 0, 295308),
    (24960, 'standard', False, 48000, 0, 925080),
    (11025, 'fast', True, 4800, 6657, 489856),
    (11025, 'fast', True, 48000, 6657, 1770860),
    (11025, 'fast', False, 4800, 0, 317432),
    (11025, 'fast', False, 48000, 0, 1076828),
    (11025, 'slow', True, 4800, 8321, 659988),
    (11025, 'slow', True, 48000, 8321, 2136604),
    (11025, 'slow', False, 4800, 0, 445012),
    (11025, 'slow', False, 48000, 0, 1269612),
    (48000, 'fast', True, 4800, 6657, 693616),
    (48000, 'fast', True, 48000, 6657, 1321976),
    (48000, 'fast', False, 4800, 0, 459672),
    (48000, 'fast', False, 48000, 0, 968224),
    (48000, 'slow', True, 4800, 8321, 612808),
    (48000, 'slow', True, 48000, 8321, 1286096),
    (48000, 'slow', False, 4800, 0, 401496),
    (48000, 'slow', False, 48000, 0, 925024),
]


def settings(profile):
    return na.Settings() if profile == "standard" else na.Settings.profile(profile)


@pytest.mark.parametrize("rate,profile", sorted(BOUNDS))
def test_decode_len_bound(rate, profile):
    got = [na.decode_len_bound(n, rate, settings(profile)) for n in (rate * 20 + 7, 9_067_017)]
    assert got == BOUNDS[(rate, profile)]


@pytest.mark.parametrize("rate,profile,sync,max_push,latency,device_bytes", GEOMETRY)
def test_stream_geometry(rate, profile, sync, max_push, latency, device_bytes):
    g = na.stream_geometry(rate, settings(profile), sync, max_push)
    assert (g["latency_work"], g["device_bytes"]) == (latency, device_bytes)
