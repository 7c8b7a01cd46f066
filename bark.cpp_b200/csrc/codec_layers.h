// The 24 kHz EnCodec's layer order, written once.  The whole-clip pipelines (codec_pipeline.cu) and the streams (codec_stream.cu) walk
// these lists with a runner that says how each layer runs on its items:
//   conv(cv, elu_in, stride)   strided_conv_1d of the current activation (ops.cpp:59-75), k = cv.k, reflect-padded
//   resblock(blk)              conv_c2(ELU conv_c1(ELU x)) + conv_sc(x), launched sc, c1, c2 (encoder.h:52-70, decoder.h:84-104)
//   convtr(cv, stride)         ELU, then strided_conv_transpose_1d (ops.cpp:77-98)
//   lstm2(w)                   the two LSTM layers, the second's input added to its output (encoder.h:98, decoder.h:72)
// The quantizer stays outside: its decode runs before the decoder's list and its encode after the encoder's, one frame at a time.
#pragma once
#include "model.h"

namespace bark {

// encoder.h:39-109: samples [1][n] -> latent [128][ceil(n / kCodecHop)]
template <class R> void encoder_layers(const CodecModel::Encoder & e, R & r) {
    r.conv(e.init, false, 1);                                            // encoder.h:49 -> [32][n]
    for (int i = 0; i < 4; i++) {                                        // encoder.h:52-83
        r.resblock(e.blk[i]);
        r.conv(e.blk[i].ds, true, kCodecRatios[3 - i]);                  // ELU -> k 2r, stride r -> [2C][ceil(L / r)]
    }
    r.lstm2(e.lstm);
    r.conv(e.final_conv, true, 1);                                       // ELU -> k7 -> latent [128][T]
}

// decoder.h:43-113: the quantizer's latent [128][T] -> waveform [1][kCodecHop T]
template <class R> void decoder_layers(const CodecModel & cm, R & r) {
    r.conv(cm.init, false, 1);                                           // [512][T]
    r.lstm2(cm.lstm);
    for (int i = 0; i < 4; i++) {
        r.convtr(cm.blk[i].us, kCodecRatios[i]);                         // ELU fused on the input; -> [C/2][L*r]
        r.resblock(cm.blk[i]);                                           // the shortcut on the raw up-sampled signal
    }
    r.conv(cm.final_conv, true, 1);                                      // ELU -> k7 -> [1][kCodecHop T]
}

}  // namespace bark
