// modes_format.cpp — the reference's human-readable message text (the default, non --raw,
// non --onlyaddr output of `dump1090 --ifile`), byte for byte: what displayModesMessage()
// (dump1090.c:1314-1450) prints plus the blank line useModesMessage() adds (dump1090.c:1813).
// Pure host code; SURVEY.md §8(f) item 1.  The wording of every line is part of the output
// format and therefore identical to the reference's; the code is ours.
#include <cstdarg>
#include <cstdio>
#include <cstring>
#include "modes_internal.h"

namespace {

struct Out {
    char *buf; size_t cap, len;
    void put(const char *fmt, ...) {
        va_list ap;
        va_start(ap, fmt);
        int n = vsnprintf(len < cap ? buf + len : nullptr, len < cap ? cap - len : 0, fmt, ap);
        va_end(ap);
        if (n > 0) len += (size_t)n;
    }
};

const char *capability_text(int ca) {
    static const char *t[8] = {
        "Level 1 (Survillance Only)", "Level 2 (DF0,4,5,11)", "Level 3 (DF0,4,5,11,20,21)",
        "Level 4 (DF0,4,5,11,20,21,24)", "Level 2+3+4 (DF0,4,5,11,20,21,24,code7 - is on ground)",
        "Level 2+3+4 (DF0,4,5,11,20,21,24,code7 - is on airborne)", "Level 2+3+4 (DF0,4,5,11,20,21,24,code7)",
        "Level 7 ???"};
    return t[ca & 7];
}

const char *flight_status_text(int fs) {
    static const char *t[8] = {
        "Normal, Airborne", "Normal, On the ground", "ALERT,  Airborne", "ALERT,  On the ground",
        "ALERT & Special Position Identification. Airborne or Ground",
        "Special Position Identification. Airborne or Ground", "Value 6 is not assigned", "Value 7 is not assigned"};
    return t[fs & 7];
}

const char *me_name(int type, int sub) {                    // dump1090.c:1060-1086
    if (type >= 1 && type <= 4) return "Aircraft Identification and Category";
    if (type >= 5 && type <= 8) return "Surface Position";
    if (type >= 9 && type <= 18) return "Airborne Position (Baro Altitude)";
    if (type == 19 && sub >= 1 && sub <= 4) return "Airborne Velocity";
    if (type >= 20 && type <= 22) return "Airborne Position (GNSS Height)";
    if (type == 23 && sub == 0) return "Test Message";
    if (type == 24 && sub == 1) return "Surface System Status";
    if (type == 28 && sub == 1) return "Extended Squitter Aircraft Status (Emergency)";
    if (type == 28 && sub == 2) return "Extended Squitter Aircraft Status (1090ES TCAS RA)";
    if (type == 29 && (sub == 0 || sub == 1)) return "Target State and Status Message";
    if (type == 31 && (sub == 0 || sub == 1)) return "Aircraft Operational Status Message";
    return "Unknown";
}

int movement_knots(int m) {                                 // dump1090.c:2056-2066
    if (m == 0) return -1;
    if (m == 1) return 0;
    if (m <= 8) return (int)((m - 2) * 0.125 + 0.125);
    if (m <= 12) return (int)((m - 9) * 0.25 + 1);
    if (m <= 38) return (int)((m - 13) * 0.5 + 2);
    if (m <= 93) return (m - 39) + 15;
    if (m <= 108) return (m - 94) * 2 + 70;
    if (m <= 123) return (m - 109) * 5 + 100;
    return 175;
}

}  // namespace

extern "C" size_t modes_format_message(const modes_message *mm, int check_crc, char *buf, size_t capacity) {
    Out o{buf, capacity, 0};
    o.put("*");
    for (int j = 0; j < mm->msgbits / 8; j++) o.put("%02x", mm->msg[j]);
    o.put(";\n");
    o.put("CRC: %06x (%s)\n", (int)mm->crc, mm->crcok ? "ok" : "wrong");
    if (mm->errorbit != -1) o.put("Single bit error fixed, bit %d\n", mm->errorbit);
    const int df = mm->msgtype;
    const char *unit = mm->unit == 1 ? "meters" : "feet";
    if (df == 0) {
        o.put("DF 0: Short Air-Air Surveillance.\n");
        o.put("  Altitude       : %d %s\n", mm->altitude, unit);
        o.put("  ICAO Address   : %02x%02x%02x\n", mm->aa1, mm->aa2, mm->aa3);
    } else if (df == 4 || df == 20) {
        o.put("DF %d: %s, Altitude Reply.\n", df, df == 4 ? "Surveillance" : "Comm-B");
        o.put("  Flight Status  : %s\n", flight_status_text(mm->fs));
        o.put("  DR             : %d\n", mm->dr);
        o.put("  UM             : %d\n", mm->um);
        o.put("  Altitude       : %d %s\n", mm->altitude, unit);
        o.put("  ICAO Address   : %02x%02x%02x\n", mm->aa1, mm->aa2, mm->aa3);
    } else if (df == 5 || df == 21) {
        o.put("DF %d: %s, Identity Reply.\n", df, df == 5 ? "Surveillance" : "Comm-B");
        o.put("  Flight Status  : %s\n", flight_status_text(mm->fs));
        o.put("  DR             : %d\n", mm->dr);
        o.put("  UM             : %d\n", mm->um);
        o.put("  Squawk         : %d\n", mm->identity);
        o.put("  ICAO Address   : %02x%02x%02x\n", mm->aa1, mm->aa2, mm->aa3);
    } else if (df == 11) {
        o.put("DF 11: All Call Reply.\n");
        o.put("  Capability  : %s\n", capability_text(mm->ca));
        o.put("  ICAO Address: %02x%02x%02x\n", mm->aa1, mm->aa2, mm->aa3);
    } else if (df == 17) {
        o.put("DF 17: ADS-B message.\n");
        o.put("  Capability     : %d (%s)\n", mm->ca, capability_text(mm->ca));
        o.put("  ICAO Address   : %02x%02x%02x\n", mm->aa1, mm->aa2, mm->aa3);
        o.put("  Extended Squitter  Type: %d\n", mm->metype);
        o.put("  Extended Squitter  Sub : %d\n", mm->mesub);
        o.put("  Extended Squitter  Name: %s\n", me_name(mm->metype, mm->mesub));
        const int t = mm->metype, s = mm->mesub;
        if (t >= 1 && t <= 4) {
            static const char *ac[4] = {"Aircraft Type D", "Aircraft Type C", "Aircraft Type B", "Aircraft Type A"};
            o.put("    Aircraft Type  : %s\n", ac[mm->aircraft_type & 3]);
            o.put("    Identification : %s\n", mm->flight);
        } else if (t >= 5 && t <= 8) {
            o.put("    F flag   : %s\n", mm->fflag ? "odd" : "even");
            o.put("    T flag   : %s\n", mm->tflag ? "UTC" : "non-UTC");
            o.put("    Movement : %d", mm->movement);
            if (mm->movement_valid) o.put(" (%d kt)\n", movement_knots(mm->movement));
            else o.put(" (not available)\n");
            o.put("    Track    : %d degrees", mm->ground_track);
            if (!mm->ground_track_valid) o.put(" (not valid)");
            o.put("\n");
            o.put("    Latitude : %d (not decoded)\n", mm->raw_latitude);
            o.put("    Longitude: %d (not decoded)\n", mm->raw_longitude);
        } else if (t >= 9 && t <= 18) {
            o.put("    F flag   : %s\n", mm->fflag ? "odd" : "even");
            o.put("    T flag   : %s\n", mm->tflag ? "UTC" : "non-UTC");
            o.put("    Altitude : %d feet\n", mm->altitude);
            o.put("    Latitude : %d (not decoded)\n", mm->raw_latitude);
            o.put("    Longitude: %d (not decoded)\n", mm->raw_longitude);
        } else if (t == 19 && s >= 1 && s <= 4) {
            if (s == 1 || s == 2) {
                o.put("    EW direction      : %d\n", mm->ew_dir);
                o.put("    EW velocity       : %d\n", mm->ew_velocity);
                o.put("    NS direction      : %d\n", mm->ns_dir);
                o.put("    NS velocity       : %d\n", mm->ns_velocity);
                o.put("    Vertical rate src : %d\n", mm->vert_rate_source);
                o.put("    Vertical rate sign: %d\n", mm->vert_rate_sign);
                o.put("    Vertical rate     : %d\n", mm->vert_rate);
            } else {
                o.put("    Heading status: %d", mm->heading_is_valid);
                o.put("    Heading: %d", mm->heading);
            }
        } else {
            o.put("    Unrecognized ME type: %d subtype: %d\n", t, s);
        }
    } else if (df == 18) {
        o.put("DF 18: Extended Squitter.\n");
        o.put("  Control Field  : %d\n", mm->ca);
        o.put("  ICAO Address   : %02x%02x%02x\n", mm->aa1, mm->aa2, mm->aa3);
        o.put("  Extended Squitter  Type: %d\n", mm->metype);
        o.put("  Extended Squitter  Sub : %d\n", mm->mesub);
        o.put("  Extended Squitter  Name: %s\n", me_name(mm->metype, mm->mesub));
    } else if (check_crc) {
        o.put("DF %d with good CRC received (decoding still not implemented).\n", df);
    }
    o.put("\n");
    return o.len;
}

// The raw TCP output line (port 30002), modesSendRawOutput dump1090.c:2381-2393: "*" + UPPERCASE
// hex + ";\n" (the stdout form of :1324-1326 is lowercase).
extern "C" size_t modes_format_raw_net(const modes_message *mm, char *buf, size_t capacity) {
    Out o{buf, capacity, 0};
    o.put("*");
    for (int j = 0; j < mm->msgbits / 8; j++) o.put("%02X", mm->msg[j]);
    o.put(";\n");
    return o.len;
}

// The Beast binary frame of the dump1090 descendants (their port 30005), Mode S frames only:
// 0x1a, type '2' (7 bytes) or '3' (14 bytes), 48-bit 12 MHz timestamp, signal byte, frame; every
// 0x1a after the leading one is doubled.  At 2 MHz one sample is 6 ticks of the 12 MHz clock; a
// measured arrival (modes_set_arrival) moves the timestamp by -7 .. +7 ticks.
extern "C" size_t modes_format_beast(const modes_message *mm, uint8_t *buf, size_t capacity) {
    const int nbytes = mm->msgbits == 112 ? 14 : 7;
    uint8_t body[2 + 6 + 1 + 14];
    size_t k = 0;
    body[k++] = nbytes == 14 ? '3' : '2';
    const __int128 ticks = (__int128)mm->sample_pos * 6 + (mm->arrival ? (int)mm->arrival - 8 : 0);
    const uint64_t ts = ticks < 0 ? 0 : (uint64_t)ticks & ((1ull << 48) - 1);
    for (int i = 5; i >= 0; i--) body[k++] = (uint8_t)(ts >> (8 * i));
    const int64_t s = mm->signal < 0 ? 0 : mm->signal;
    const int64_t level = (s * 255 + 32767) / 65535;
    body[k++] = (uint8_t)(level > 255 ? 255 : level);
    for (int i = 0; i < nbytes; i++) body[k++] = mm->msg[i];
    size_t len = 0;
    auto put = [&](uint8_t b) { if (len < capacity) buf[len] = b; len++; };
    put(0x1a);
    for (size_t i = 0; i < k; i++) {
        put(body[i]);
        if (body[i] == 0x1a) put(0x1a);
    }
    return len;
}

// The raw TCP input line (port 30001), the parsing half of decodeHexMessage dump1090.c:2472-2497:
// surrounding white space ignored, "*" ... ";" required, at most 28 hex digits, any non-hex digit
// (or an odd digit count, which makes the reference pair a digit with ';') discards the line.
// Returns the number of frame bytes written (0..14) or -1 if the reference discards the line.
// Bytes the line does not supply are zeroed (the reference leaves them uninitialised).
extern "C" int modes_parse_hex_line(const char *line, uint8_t msg[14]) {
    auto is_space = [](unsigned char c) { return c == ' ' || (c >= '\t' && c <= '\r'); };
    auto hexval = [](unsigned char c) -> int {
        if (c >= '0' && c <= '9') return c - '0';
        c |= 0x20;
        if (c >= 'a' && c <= 'f') return c - 'a' + 10;
        return -1;
    };
    std::memset(msg, 0, 14);
    size_t l = std::strlen(line);
    while (l && is_space((unsigned char)line[l - 1])) l--;
    while (l && is_space((unsigned char)*line)) { line++; l--; }
    if (l < 2 || line[0] != '*' || line[l - 1] != ';') return -1;
    line++; l -= 2;
    if (l > 28) return -1;
    for (size_t j = 0; j < l; j += 2) {
        const int hi = hexval((unsigned char)line[j]);
        const int lo = j + 1 < l ? hexval((unsigned char)line[j + 1]) : -1;
        if (hi < 0 || lo < 0) return -1;
        msg[j / 2] = (uint8_t)((hi << 4) | lo);
    }
    return (int)(l / 2);
}
