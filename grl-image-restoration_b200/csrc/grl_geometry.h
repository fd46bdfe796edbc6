// grl_geometry.h -- closed-form index arithmetic shared by host code and every attention kernel.
//
// The reference builds int64 index tensors and -100 masks on the CPU (models/common/ops.py) and
// keeps ~1.5 GB of them as module buffers (models/networks/grl.py:386-429).  Here they are O(1)
// functions evaluated in registers; the grl_*_host() functions expand them into tensors so the tests can
// check them bit-exactly against the reference's golden digests.
#pragma once
#include <stdint.h>

#include "../../include/grl_b200.h"
#include "grl_hd.h"

namespace grl {

struct Tok {
  int r, c;  // coordinates in the ROLLED grid
  int y, x;  // coordinates in the un-rolled (memory) grid
  int ih, iw;  // coordinates inside the window
};

// Token n of window (wr, wc):  rolled position, then un-roll  R[r,c] = X[(r+s) mod H]  (torch.roll by -s,
// mixed_attn_block_efficient.py:141-143,:236-241) and window_partition's row-major order (ops.py:45-53).
GRL_HD Tok locate(const GrlGrid& g, int wr, int wc, int n) {
  Tok t;
  t.ih = n / g.ww;
  t.iw = n - t.ih * g.ww;
  t.r = wr * g.wh + t.ih;
  t.c = wc * g.ww + t.iw;
  t.y = t.r + g.sh;
  if (t.y >= g.H) t.y -= g.H;
  t.x = t.c + g.sw;
  if (t.x >= g.W) t.x -= g.W;
  return t;
}

// Region id of a rolled position: ops.py:76-99 (_fill_window) as a closed form.  Only (in)equality of two
// ids inside one window is ever used (ops.py:120-125,:148-155), and that matches the reference's
// sequential-slice construction for every shift, including the degenerate shift == 0 (SURVEY.md A.6).
GRL_HD int region_id(const GrlGrid& g, int r, int c) {
  int a = (r >= g.H - g.wh) + (g.sh > 0 && r >= g.H - g.sh);
  int b = (c >= g.W - g.ww) + (g.sw > 0 && c >= g.W - g.sw);
  return 3 * a + b;
}

// Relative-position index between a query token (qh,qw) of a (.., qww)-wide window and a key token (kh,kw)
// of a (kwh x kww) window: get_relative_position_index_simple + coords_diff_odd (ops.py:308-316,:352-375).
// window->anchor: q = window token, k = anchor; anchor->window: q = anchor, k = window token.
GRL_HD int rel_index(int qh, int qw, int kh, int kw, int qww, int kwh, int kww) {
  return (qh - kh + kwh - 1) * (qww + kww - 1) + (qw - kw + kww - 1);
}

GRL_HD int windows_per_image(const GrlGrid& g) { return (g.H / g.wh) * (g.W / g.ww); }

// Host check of a grid before anything above is evaluated on it; `what` names the caller in the message.
int fail(int code, const char* fmt, ...);  // grl_common.cuh
inline int check_grid(const GrlGrid& g, const char* what) {
  if (!(g.H > 0 && g.W > 0 && g.wh > 0 && g.ww > 0)) return fail(GRL_ERR_INVALID, "%s: empty grid", what);
  if (!(g.H % g.wh == 0 && g.W % g.ww == 0))
    return fail(GRL_ERR_INVALID, "%s: grid %dx%d is not a multiple of the window %dx%d", what, g.H, g.W, g.wh, g.ww);
  if (!(g.sh >= 0 && g.sh < g.H && g.sw >= 0 && g.sw < g.W && g.sh <= g.wh && g.sw <= g.ww))
    return fail(GRL_ERR_INVALID, "%s: bad shift (%d,%d)", what, g.sh, g.sw);
  return GRL_OK;
}

// The 8 dihedral views of augment_img_tensor4 (utils/utils_bsr/utils_image.py:444-460) as closed forms.  The mode's
// bits are: 1 = transpose (the view is W x H), 2 = flip the source rows, 4 = flip the source columns:
//   0 identity, 1 transpose, 2 flip(H), 3 rot90 k=3, 4 flip(W), 5 rot90 k=1, 6 rot180, 7 anti-transpose.
struct Pix {
  int y, x;
};
GRL_HD bool d8_transposes(int mode) { return (mode & 1) != 0; }

// Source pixel in the (H x W) image of position (y, x) of view `mode` (which is H x W, or W x H when it transposes).
GRL_HD Pix d8_src(int mode, int y, int x, int H, int W) {
  const int r = (mode & 1) ? x : y, c = (mode & 1) ? y : x;
  return {(mode & 2) ? H - 1 - r : r, (mode & 4) ? W - 1 - c : c};
}

// The way back: position in view `mode` of pixel (y, x) of the (H x W) image, i.e. d8_src(mode, .)^-1.  Every mode but 3
// and 5 is its own inverse; for those two this is view 8 - mode applied to the view.
GRL_HD Pix d8_inv(int mode, int y, int x, int H, int W) {
  const int r = (mode & 2) ? H - 1 - y : y, c = (mode & 4) ? W - 1 - x : x;
  return (mode & 1) ? Pix{c, r} : Pix{r, c};
}

}  // namespace grl
