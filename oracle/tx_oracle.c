/*
 * tx_oracle.c -- TEST INFRASTRUCTURE: the reference's transmit loop over input events, and the host
 * build of the product's encoders.
 *
 * fsk_oracle.c restates the tone generator and fsk_transmit_frame for a whole block of data words
 * (orc_tx_words).  A transmitter fed in pieces also needs the loop around them: the leader only when
 * the carrier was off, the sync preamble again after an idle timeout, the idle tone, the trailer at
 * end of input.  This file includes fsk_oracle.c for its (static) tone generator and frame writer
 * and adds that loop, so the two share every sample-level statement.  The encoders come from
 * minimodem_b200/csrc/fsk_b200_decode_core.h (fsk_enc_byte), the very source the tx kernel compiles,
 * so that the CPU tests can hold them against the reference's databits_encode_ascii8 / baudot_encode
 * in oracle/_ref/libfsk_ref.so.  Built by tests/txorc.py; nothing in the product links it.
 */
#include "fsk_oracle.c"
#include "../minimodem_b200/csrc/fsk_b200_decode_core.h"

/* events[i] = 0..255: a byte read from stdin; ORC_TX_IDLE: a select() timeout (the writer of the
 * pipe paused for idle_carrier_usec, src/minimodem.c:176-192) */
#define ORC_TX_IDLE (-1)
/* the databits encoder, words-level: at most 2 words per byte */
typedef unsigned (*orc_encode_fn)(void *ctx, unsigned char byte, unsigned *words);

/* fsk_transmit_stdin, src/minimodem.c:114-250, non-interactive, over the events; after the last
 * event comes end of file: the trailer when transmitting (:246-249, :59-74).  Returns the samples
 * produced (the first out_cap stored). */
size_t orc_tx_events(const orc_tx_config *cfg, const int *events, size_t nevents, orc_encode_fn encode,
	void *ctx, float *out, size_t out_cap)
{
    struct tonegen g;
    tonegen_init(&g, cfg, out, out_cap);
    struct tx_lengths L = tx_lengths(cfg);
    const size_t sample_rate = (size_t)cfg->sample_rate;
    const unsigned idle_carrier_usec = 1000000 / 25;			/* :155 */
    const float idle_f = cfg->invert_start_stop ? cfg->f_space : cfg->f_mark;
    int tx_transmitting = 0;
    for (size_t e = 0; e < nevents; e++) {
	if (events[e] == ORC_TX_IDLE) {					/* :230-237 */
	    tx_transmitting = 1;
	    tonegen_tone(&g, idle_f, idle_carrier_usec * sample_rate / 1000000);
	    continue;
	}
	unsigned words[2];
	const unsigned nwords = encode(ctx, (unsigned char)events[e], words);	/* :205 */
	if (!tx_transmitting) {						/* :207-213 */
	    tx_transmitting = 1;
	    for (int j = 0; j < cfg->leader_bits; j++)
		tonegen_tone(&g, idle_f, L.bit);
	}
	if (tx_transmitting < 2) {					/* :214-222 */
	    tx_transmitting = 2;
	    for (unsigned j = 0; j < cfg->do_tx_sync_bytes; j++)
		tx_frame(&g, cfg, L, cfg->sync_byte, 0);
	}
	for (unsigned j = 0; j < nwords; j++)				/* :225-228 */
	    tx_frame(&g, cfg, L, words[j], cfg->msb_first);
    }
    if (tx_transmitting)						/* :246-249 */
	for (int j = 0; j < cfg->trailer_bits; j++)
	    tonegen_tone(&g, cfg->f_mark, L.bit);
    size_t n = g.n;
    tonegen_free(&g);
    return n;
}

/* the product's encoders (fsk_enc_byte), host build: ctx = { kind, charset } with the charset carried
 * from call to call; fits orc_tx_events' orc_encode_fn */
typedef struct orc_encoder { int kind; uint32_t charset; } orc_encoder;

unsigned orc_encode_byte(void *ctx, unsigned char byte, unsigned *words)
{
    orc_encoder *e = (orc_encoder *)ctx;
    uint32_t w[2];
    unsigned n = fsk_enc_byte(e->kind, &e->charset, byte, w);
    for (unsigned i = 0; i < n; i++)
	words[i] = w[i];
    return n;
}
