// Option string of the GPUJPEG compress module, shared by the two builds of the module (host/video_compress.cpp against the mirror types,
// module/ug_module.cpp against UltraGrid's own headers).  Grammar and meaning of state_video_compress_gpujpeg::parse_fmt,
// src/video_compress/gpujpeg.cpp:371-424:
//     <quality>[:<restart interval>] positionally, or quality=<n> (here also q=<n>), restart=<n>, interleaved, Y601 | Y601full | Y709 | RGB,
//     subsampling=<444|422|420>, alpha; plus lanes=<n> (addition of this library: frames in flight per device).
// This module stores the input as it comes (RGB input -> RGB, 4:4:4; UYVY input -> BT.709 YCbCr, 4:2:2; I420 input -> BT.709 YCbCr, 4:2:0 - the
// reference's own defaults, :295-305, :332; RGBA input with `alpha` -> R G B A, four components 1x1, :227-236,316-328): an internal colour space or a
// subsampling other than the input's own is refused when the first frame
// shows the input format (check_against_input), with a message instead of a silently different stream.  The encoder itself can also convert
// RGB to YCbCr and subsample chroma (ugb200_jpeg_encode_into_ex); opening those options here is a change of this policy only.
#pragma once
#include <cctype>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <strings.h>

enum class jpeg_input { UYVY, RGB, I420, RGBA };  // the encoder input formats (RGBA: only with `alpha`, read in place)

struct gpujpeg_opts {
        int quality = -1;           // -1: encoder default (gpujpeg_set_default_parameters: 75)
        int restart_interval = 0;   // 0: default for the input format
        bool interleaved = false;   // m_force_interleaved
        int internal_cs = 0;        // 0 unset, 1 Y601, 2 Y601full, 3 Y709, 4 RGB
        int subsampling = 0;        // 0 auto, else 444 / 422 / 420
        bool alpha = false;         // RGBA input: four components (the alpha channel kept)
        int lanes = 3;
        bool help = false;

        /// @returns false on a malformed option (message on stderr)
        bool parse(const char *opts)
        {
                std::string o = opts ? opts : "";
                size_t pos = 0;
                int idx = 0;
                while (pos <= o.size() && !o.empty()) {
                        size_t end = o.find(':', pos);
                        end = end == std::string::npos ? o.size() : end;
                        const std::string t = o.substr(pos, end - pos);
                        pos = end + 1;
                        if (t.empty()) {
                                if (pos > o.size()) {
                                        break;
                                }
                                continue;
                        }
                        const char *tok = t.c_str();
                        const char *eq = strchr(tok, '=');
                        if (isdigit((unsigned char) tok[0]) && idx == 0) {
                                quality = atoi(tok);
                                if (quality <= 0 || quality > 100) {
                                        fprintf(stderr, "[GPUJPEG] Error: Quality should be in interval [1-100]!\n");
                                        return false;
                                }
                        } else if (isdigit((unsigned char) tok[0]) && idx == 1) {
                                restart_interval = atoi(tok);
                        } else if (t == "help") {
                                help = true;
                        } else if (eq && (strncasecmp(tok, "quality=", 8) == 0 || strncasecmp(tok, "q=", 2) == 0)) {
                                quality = atoi(eq + 1);
                                if (quality <= 0 || quality > 100) {
                                        fprintf(stderr, "[GPUJPEG] Error: Quality should be in interval [1-100]!\n");
                                        return false;
                                }
                        } else if (eq && strncasecmp(tok, "restart=", 8) == 0) {
                                restart_interval = atoi(eq + 1);
                                if (restart_interval < 0) {
                                        fprintf(stderr, "[GPUJPEG] Error: Restart interval should be non-negative!\n");
                                        return false;
                                }
                        } else if (strncasecmp(tok, "interleaved", 11) == 0) {
                                interleaved = true;
                        } else if (strcasecmp(tok, "Y601") == 0) {
                                internal_cs = 1;
                        } else if (strcasecmp(tok, "Y601full") == 0) {
                                internal_cs = 2;
                        } else if (strcasecmp(tok, "Y709") == 0) {
                                internal_cs = 3;
                        } else if (strcasecmp(tok, "RGB") == 0) {
                                internal_cs = 4;
                        } else if (eq && strncasecmp(tok, "subsampling=", 12) == 0) {
                                subsampling = atoi(eq + 1);
                                if (subsampling != 444 && subsampling != 422 && subsampling != 420) {
                                        fprintf(stderr, "[GPUJPEG] Error: subsampling must be 444, 422 or 420!\n");
                                        return false;
                                }
                        } else if (t == "alpha") {
                                alpha = true;
                        } else if (eq && strncasecmp(tok, "lanes=", 6) == 0) {
                                lanes = atoi(eq + 1);
                                if (lanes < 1 || lanes > 8) {
                                        fprintf(stderr, "[GPUJPEG] lanes must be 1..8\n");
                                        return false;
                                }
                        } else {
                                fprintf(stderr, "[GPUJPEG] Unknown configuration parameter or a missing value: %s\n", tok);
                                return false;
                        }
                        ++idx;
                }
                return true;
        }

        static void usage()
        {
                printf("GPUJPEG usage:\n\t-c GPUJPEG[:<quality>[:<restart_interval>]][:quality=<q>][:restart=<n>][:interleaved][:RGB|Y709][:subsampling=<444|422|420>][:alpha][:lanes=<n>]\n"
                       "\twhere\n\t\tinterleaved - one scan for RGB and RGBA input too (default: one scan per component)\n"
                       "\t\tRGB|Y709 - must name the colour space the input already has (no transform inside the codec)\n"
                       "\t\tsubsampling - must name the input's own: 444 for RGB, 422 for UYVY, 420 for I420 (I420 frames are encoded as they are)\n"
                       "\t\talpha - RGBA input is encoded with its alpha channel as a fourth component (subsampling 4:4:4:4; RGB colour space only)\n"
                       "\t\tlanes - frames in flight per CUDA device (default 3)\n");
        }

        /// the options against the encoder input format: what needs a transform inside the codec is refused
        bool check_against_input(jpeg_input in) const
        {
                if (in == jpeg_input::RGBA) {  // `alpha` with RGBA frames: R G B A as stored, every component 1x1
                        if (internal_cs != 0 && internal_cs != 4) {
                                fprintf(stderr, "[GPUJPEG] alpha: RGBA input is stored as R G B A; the requested internal colour space needs a colour transform inside the codec\n");
                                return false;
                        }
                        if (subsampling != 0 && subsampling != 444) {
                                fprintf(stderr, "[GPUJPEG] alpha: subsampling=%d needs resampling inside the codec; RGBA input is stored as 4:4:4:4\n", subsampling);
                                return false;
                        }
                        return true;
                }
                const char *name = in == jpeg_input::RGB ? "RGB" : in == jpeg_input::UYVY ? "UYVY" : "I420";
                if (internal_cs != 0 && internal_cs != (in == jpeg_input::RGB ? 4 : 3)) {
                        fprintf(stderr, "[GPUJPEG] the requested internal colour space needs a colour transform inside the codec; this encoder stores %s input as %s\n",
                                name, in == jpeg_input::RGB ? "RGB" : "BT.709 YCbCr");
                        return false;
                }
                const int native = in == jpeg_input::RGB ? 444 : in == jpeg_input::UYVY ? 422 : 420;
                if (subsampling != 0 && subsampling != native) {
                        fprintf(stderr, "[GPUJPEG] subsampling=%d needs resampling inside the codec; %s input is stored as 4:%s\n", subsampling, name,
                                native == 444 ? "4:4" : native == 422 ? "2:2" : "2:0");
                        return false;
                }
                if (alpha) {
                        fprintf(stderr, "[GPUJPEG] Requested alpha encode but the input is not RGBA; alpha is dropped\n");
                }
                return true;
        }
};
