/*
 * fsk_b200_decode_core.h -- N1: data words -> output bytes, the reference's
 * databits decoders with their file-static state made per-stream.
 *
 * One source for two builds: nvcc compiles it into k_decode (one thread per stream walks that
 * stream's frame records); gcc compiles it into the test harness (oracle/decode_oracle.c), where
 * it is checked byte for byte against the unmodified reference decoders.  Nothing in the
 * product calls the host build.
 *
 * Follows (behaviour, not text):
 *   ascii   src/databits_ascii.c:35-44        one byte per word
 *   binary  src/databits_binary.c:29-41       n_data_bits chars '0'/'1', LSB first, then '\n'
 *   baudot  src/databits_baudot.c:30-40, src/baudot.c:33-70,187-243   ITA2, US figures,
 *           unshift-on-space; LTRS/FIGS select the case and print nothing
 *   callerid src/databits_callerid.c:38-209   SDMF/MDMF collector and formatter, including
 *           that a message is complete one byte early (the checksum byte is never collected,
 *           :185-186), that the 256-byte message buffer is never cleared, and that a bad
 *           MDMF field discards the fields printed before it (:62-71)
 *   uic     src/databits_uic.c:29-74, src/uic_codes.c:23-68   one text line per 39-bit word
 *
 * and the transmitter's two encoders (bytes -> data words), compiled into the tx kernel and, for the
 * tests, by gcc into oracle/tx_oracle.c:
 *   ascii8  src/databits_ascii.c:28-33        the byte, sign-extended as a char
 *   baudot  src/baudot.c:258-310              ITA2 from the decoder's columns, shift codes,
 *           unshift-on-space, non-encodable characters skipped
 */
#ifndef FSK_B200_DECODE_CORE_H
#define FSK_B200_DECODE_CORE_H

#include <stdint.h>
#include "fsk_b200.h"

#ifdef __CUDACC__
#define FSK_HD __host__ __device__ __forceinline__
#else
#define FSK_HD static inline
#endif

/* output of one stream: every byte is counted, the first `cap` are stored */
typedef struct fsk_dec_sink {
    uint8_t *out;
    uint32_t cap, n;
} fsk_dec_sink;

FSK_HD void fsk_dec_put(fsk_dec_sink *k, unsigned int c)
{
    if (k->n < k->cap)
	k->out[k->n] = (uint8_t)c;
    k->n++;
}

/* printf("%s") of a literal */
FSK_HD void fsk_dec_puts(fsk_dec_sink *k, const char *s)
{
    while (*s)
	fsk_dec_put(k, (unsigned char)*s++);
}

/* printf("%-6s ") of a literal: left-justified in 6 columns, then a blank */
FSK_HD void fsk_dec_put_label(fsk_dec_sink *k, const char *s)
{
    unsigned int w = 0;
    while (*s) {
	fsk_dec_put(k, (unsigned char)*s++);
	w++;
    }
    for (; w < 6; w++)
	fsk_dec_put(k, ' ');
    fsk_dec_put(k, ' ');
}

/* printf("%.*s") out of the message buffer: at most `prec` bytes (negative: no limit), stops at
 * a NUL; bytes past the 256-byte buffer read as NUL (the reference would read whatever
 * follows its static array) */
FSK_HD void fsk_dec_put_field(fsk_dec_sink *k, const uint8_t *buf, unsigned int at, int prec)
{
    for (unsigned int i = 0; prec < 0 || i < (unsigned int)prec; i++) {
	if (at + i >= 256u || buf[at + i] == 0)
	    break;
	fsk_dec_put(k, buf[at + i]);
    }
}

/* ------------------------------------------------------------------------ */
/* Baudot (ITA2)                                                            */
/* ------------------------------------------------------------------------ */

/* column 0: letters; column 1: U.S. figures (src/baudot.c:33-70; 0x07 = BELL).  '_', '^' and '%'
 * are the reference's debugging marks for NUL and the two shift codes. */
FSK_HD unsigned int fsk_dec_baudot_char(unsigned int code, unsigned int figs)
{
    const char *ltrs = "_E\nA SIU\rDRJNFCKTZLWHYPQOBG%MXV%";
    const char *usfg = "^3\n- \a87\r$4',!:(5\")2#6019?&%./;%";
    return (unsigned char)(figs ? usfg[code & 31u] : ltrs[code & 31u]);
}

FSK_HD void fsk_dec_baudot(fsk_b200_decoder_state *st, unsigned int code, fsk_dec_sink *k)
{
    code &= 0x1fu;					/* src/databits_baudot.c:38 */
    if (code == 0x1bu) {				/* FIGS, src/baudot.c:224-226 */
	st->baudot_charset = 2;
	return;
    }
    if (code == 0x1fu) {				/* LTRS, :227-229 */
	st->baudot_charset = 1;
	return;
    }
    if (code == 0x04u)					/* unshift on space, :230-232 (baudot_usos = 1) */
	st->baudot_charset = 1;
    fsk_dec_put(k, fsk_dec_baudot_char(code, st->baudot_charset != 1u));	/* :234-241 */
}

/* ------------------------------------------------------------------------ */
/* Caller-ID (SDMF / MDMF)                                                  */
/* ------------------------------------------------------------------------ */

FSK_HD const char *fsk_dec_cid_label(unsigned int datatype)
{
    switch (datatype) {					/* src/databits_callerid.c:38-42 */
	case 1: return "Time:";
	case 2: case 4: return "Phone:";
	case 7: case 8: return "Name:";
	case 0: return "unknown0:";
	case 3: return "unknown3:";
	case 5: return "unknown5:";
	default: return "unknown6:";
    }
}

/* "%.2s/%.2s %.2s:%.2s\n" */
FSK_HD void fsk_dec_cid_datetime(fsk_dec_sink *k, const uint8_t *buf, unsigned int m)
{
    fsk_dec_put_field(k, buf, m + 0, 2);
    fsk_dec_put(k, '/');
    fsk_dec_put_field(k, buf, m + 2, 2);
    fsk_dec_put(k, ' ');
    fsk_dec_put_field(k, buf, m + 4, 2);
    fsk_dec_put(k, ':');
    fsk_dec_put_field(k, buf, m + 6, 2);
    fsk_dec_put(k, '\n');
}

/* "%.3s-%.3s-%.4s\n" */
FSK_HD void fsk_dec_cid_phone10(fsk_dec_sink *k, const uint8_t *buf, unsigned int m)
{
    fsk_dec_put_field(k, buf, m + 0, 3);
    fsk_dec_put(k, '-');
    fsk_dec_put_field(k, buf, m + 3, 3);
    fsk_dec_put(k, '-');
    fsk_dec_put_field(k, buf, m + 6, 4);
    fsk_dec_put(k, '\n');
}

/* src/databits_callerid.c:50-124; returns 0 when the datastream is bad (the caller then drops
 * what this function printed) */
FSK_HD int fsk_dec_cid_mdmf(const uint8_t *buf, fsk_dec_sink *k)
{
    const unsigned int msglen = buf[1];
    unsigned int m = 2, i = 0;
    while (i < msglen) {
	/* m can run past the buffer only through reads the reference would make past its array */
	const unsigned int datatype = m < 256u ? buf[m] : 0u;
	m++;
	if (datatype > 8u)				/* :62-65 */
	    return 0;
	const unsigned int datalen = m < 256u ? buf[m] : 0u;
	m++;
	if (m + 2u + datalen >= 256u)			/* :68-71 */
	    return 0;
	fsk_dec_put_label(k, fsk_dec_cid_label(datatype));	/* :75-76 */
	int plain = 0;
	switch (datatype) {
	    case 1:					/* :81-84 */
		fsk_dec_cid_datetime(k, buf, m);
		break;
	    case 2:					/* :85-92: ten digits, else printed like a name */
		if (datalen == 10u)
		    fsk_dec_cid_phone10(k, buf, m);
		else
		    plain = 1;
		break;
	    case 7:					/* :93-96 */
		plain = 1;
		break;
	    case 4:					/* :97-106 */
	    case 8:
		if (datalen == 1u && buf[m] == 'O')
		    fsk_dec_puts(k, "[N/A]\n");
		else if (datalen == 1u && buf[m] == 'P')
		    fsk_dec_puts(k, "[blocked]\n");
		break;
	    default:
		break;
	}
	if (plain) {					/* :111-112 */
	    fsk_dec_put_field(k, buf, m, (int)datalen);
	    fsk_dec_put(k, '\n');
	}
	m += datalen;					/* :114-115 */
	i += datalen + 2u;
    }
    return 1;
}

/* src/databits_callerid.c:127-153 */
FSK_HD void fsk_dec_cid_sdmf(const uint8_t *buf, fsk_dec_sink *k)
{
    const unsigned int msglen = buf[1];
    fsk_dec_put_label(k, "Time:");
    fsk_dec_cid_datetime(k, buf, 2);
    fsk_dec_put_label(k, "Phone:");
    const unsigned int datalen = msglen - 8u;		/* unsigned, as there: wraps below 8 */
    if (datalen == 10u)
	fsk_dec_cid_phone10(k, buf, 10);
    else {
	fsk_dec_put_field(k, buf, 10, (int)datalen);	/* a wrapped length is a negative precision: no limit */
	fsk_dec_put(k, '\n');
    }
}

FSK_HD void fsk_dec_callerid(fsk_b200_decoder_state *st, unsigned long long word, fsk_dec_sink *k)
{
    if (st->cid_msgtype == 0) {				/* :171-180: wait for a message type byte */
	if (word == 0x80ull)
	    st->cid_msgtype = 0x80;
	else if (word == 0x04ull)
	    st->cid_msgtype = 0x04;
	else
	    return;
	st->cid_buf[st->cid_ndata++] = (uint8_t)word;
	return;
    }
    if (st->cid_ndata >= 256u) {			/* :182-185 */
	st->cid_msgtype = 0;
	st->cid_ndata = 0;
	return;
    }
    st->cid_buf[st->cid_ndata++] = (uint8_t)word;	/* :187 */
    if (st->cid_ndata < (unsigned int)st->cid_buf[1] + 2u)	/* :192-194 */
	return;
    fsk_dec_puts(k, "CALLER-ID\n");			/* :202 */
    if (st->cid_msgtype == 0x80u) {
	const uint32_t mark = k->n;
	if (!fsk_dec_cid_mdmf(st->cid_buf, k))
	    k->n = mark;				/* the bad message's fields are not counted */
    } else
	fsk_dec_cid_sdmf(st->cid_buf, k);
    st->cid_msgtype = 0;				/* :212 */
    st->cid_ndata = 0;
}

/* ------------------------------------------------------------------------ */
/* UIC-751-3                                                                */
/* ------------------------------------------------------------------------ */

FSK_HD const char *fsk_dec_uic_meaning(unsigned int code, int train_to_ground)
{
    if (!train_to_ground) {				/* src/uic_codes.c:23-34 */
	switch (code) {
	    case 0x00: return "Test";
	    case 0x02: return "Run slower";
	    case 0x03: return "Extension of telegram";
	    case 0x04: return "Run faster";
	    case 0x06: return "Written order";
	    case 0x08: return "Speech";
	    case 0x09: return "Emergency stop";
	    case 0x0C: return "Announcem. by loudspeaker";
	    case 0x55: return "Idle";
	    default: return "Unknown";
	}
    }
    switch (code) {					/* :36-45 */
	case 0x08: return "Communic. desired";
	case 0x0A: return "Acknowl. of order";
	case 0x06: return "Advice";
	case 0x00: return "Test";
	case 0x09: return "Train staff wish to comm.";
	case 0x0C: return "Telephone link desired";
	case 0x03: return "Extension of telegram";
	default: return "Unknown";
    }
}

FSK_HD void fsk_dec_put_hex1(fsk_dec_sink *k, unsigned int v)
{
    v &= 15u;
    fsk_dec_put(k, v < 10u ? '0' + v : 'A' + (v - 10u));
}

/* src/databits_uic.c:29-52: "Train ID: %X%X%X%X%X%X - Message: %02X (%s)\n" */
FSK_HD void fsk_dec_uic(unsigned long long word, int train_to_ground, fsk_dec_sink *k)
{
    unsigned int code = 0;				/* bit_reverse(bit_window(word, 24, 8), 8) */
    for (unsigned int b = 0; b < 8u; b++)
	code = (code << 1) | (unsigned int)((word >> (24u + b)) & 1ull);
    fsk_dec_puts(k, "Train ID: ");
    for (unsigned int d = 0; d < 6u; d++)
	fsk_dec_put_hex1(k, (unsigned int)(word >> (4u * d)));
    fsk_dec_puts(k, " - Message: ");
    fsk_dec_put_hex1(k, code >> 4);
    fsk_dec_put_hex1(k, code);
    fsk_dec_puts(k, " (");
    fsk_dec_puts(k, fsk_dec_uic_meaning(code, train_to_ground));
    fsk_dec_puts(k, ")\n");
}

/* ------------------------------------------------------------------------ */
/* the decoder interface of src/databits.h:51-53, per stream                */
/* ------------------------------------------------------------------------ */

/* databits_decode(0, 0, 0, 0): the reset at carrier acquire, src/minimodem.c:1351 */
FSK_HD void fsk_dec_reset(int kind, fsk_b200_decoder_state *st)
{
    if (kind == FSK_B200_DECODE_BAUDOT)
	st->baudot_charset = 1;				/* src/baudot.c:207-211 */
    else if (kind == FSK_B200_DECODE_CALLERID) {
	st->cid_msgtype = 0;				/* src/databits_callerid.c:156-161 */
	st->cid_ndata = 0;
    }
}

FSK_HD void fsk_dec_word(int kind, unsigned int n_data_bits, fsk_b200_decoder_state *st,
	unsigned long long word, fsk_dec_sink *k)
{
    switch (kind) {
	case FSK_B200_DECODE_ASCII:
	    fsk_dec_put(k, (unsigned int)(word & 0xffull));
	    break;
	case FSK_B200_DECODE_BINARY:
	    for (unsigned int j = 0; j < n_data_bits; j++)
		fsk_dec_put(k, '0' + (unsigned int)((word >> j) & 1ull));
	    fsk_dec_put(k, '\n');
	    break;
	case FSK_B200_DECODE_BAUDOT:
	    fsk_dec_baudot(st, (unsigned int)word, k);
	    break;
	case FSK_B200_DECODE_CALLERID:
	    fsk_dec_callerid(st, word, k);
	    break;
	case FSK_B200_DECODE_UIC_GROUND:
	    fsk_dec_uic(word, 0, k);
	    break;
	case FSK_B200_DECODE_UIC_TRAIN:
	    fsk_dec_uic(word, 1, k);
	    break;
	default:
	    break;
    }
}

/* One frame record of a stream, as the rx loop treats it (src/minimodem.c:1351, :1415-1446):
 * reset on the record that acquired the carrier, prev-stop chop + bit_window (+ bit_reverse),
 * sync-byte suppression, decode.  `rec` = the 5 words of an fsk_b200_frame. */
FSK_HD void fsk_dec_record(int kind, unsigned int shift, unsigned int n_data_bits, int msb_first,
	int do_rx_sync, unsigned long long sync_byte, fsk_b200_decoder_state *st,
	const uint32_t *rec, fsk_dec_sink *k)
{
    if (rec[4] == FSK_B200_FRAME_REPORT)
	return;						/* a carrier-session report, not a frame */
    if (rec[4] & FSK_B200_FRAME_ACQUIRED)
	fsk_dec_reset(kind, st);
    unsigned long long bits = ((unsigned long long)rec[1] << 32) | rec[0];
    bits >>= shift;
    if (n_data_bits < 64u)
	bits &= (1ull << n_data_bits) - 1ull;
    if (msb_first) {					/* bit_reverse keeps 32 bits (src/databits.h:21-33) */
	unsigned int r = 0;
	for (unsigned int b = 0; b < n_data_bits; b++)
	    r = (r << 1) | (unsigned int)((bits >> b) & 1ull);
	bits = r;
    }
    if (do_rx_sync && bits == sync_byte)		/* :1436-1439 */
	return;
    fsk_dec_word(kind, n_data_bits, st, bits, k);
}

/* ------------------------------------------------------------------------ */
/* the databits encoders of the transmitter (src/databits.h:48-65)          */
/* ------------------------------------------------------------------------ */

/* databits_encode_ascii8, src/databits_ascii.c:28-33: the byte as a (signed) char, so that
 * bytes >= 0x80 are sign-extended into the word */
FSK_HD uint32_t fsk_enc_ascii8(unsigned int byte)
{
    return (uint32_t)(int32_t)(int8_t)(uint8_t)byte;
}

/* toupper() of the C locale on a char value (-128..127) */
FSK_HD int fsk_enc_toupper(int c)
{
    return c >= 'a' && c <= 'z' ? c - ('a' - 'A') : c;
}

/* Which charsets hold ASCII character c (0 <= c < 0x60) and under which code, read off the
 * decoder's columns (fsk_dec_baudot_char): (mask << 8) | code, mask bit 0 = LTRS, bit 1 = U.S.
 * FIGS, 0 = not encodable.  Code 0 is NUL in both columns (the decoder prints '_' / '^' for it),
 * the two shift codes carry no character.  One deviation from the plain inversion is the
 * reference's own: its encoder sends '+' as 0x12 in FIGS (')' in the U.S. column; '+' is the
 * CCITT No. 2 figure of 0x11), src/baudot.c baudot_encode_table. */
FSK_HD unsigned int fsk_enc_baudot_entry(int c)
{
    if (c == '+')
	return (2u << 8) | 0x12u;
    unsigned int mask = 0, code = 0;
    for (unsigned int k = 0; k < 32u; k++) {
	if (k == 0x1bu || k == 0x1fu)
	    continue;
	const int l = k ? (int)fsk_dec_baudot_char(k, 0) : 0;
	const int f = k ? (int)fsk_dec_baudot_char(k, 1) : 0;
	if (c == l) {
	    mask |= 1u;
	    code = k;
	}
	if (c == f) {
	    mask |= 2u;
	    code = k;
	}
    }
    return (mask << 8) | code;
}

/* baudot_encode, src/baudot.c:258-310 (baudot_usos = 1), with the file-static baudot_charset
 * held in *charset (0 unknown, 1 LTRS, 2 FIGS).  c: toupper() of the char value, entry:
 * fsk_enc_baudot_entry(c) when 0 <= c < 0x60 (anything, otherwise).  Returns the number of
 * words stored (0, 1 or 2): a shift code first when the character is not in the current
 * charset, then the character's code. */
FSK_HD unsigned int fsk_enc_baudot_with(uint32_t *charset, int c, unsigned int entry, uint32_t *words)
{
    if (c >= 0x60 || c < 0)				/* :263-267 */
	return 0;
    const unsigned int mask = entry >> 8;
    unsigned int shift = 0;
    if ((*charset & mask) == 0) {			/* :277-294 */
	if (mask == 0)
	    return 0;
	if (*charset == 0)
	    *charset = 1;
	if (mask != 3u)
	    *charset = mask;
	shift = *charset == 1u ? 0x1Fu : 0x1Bu;
    }
    if (c == ' ')					/* :305-306 */
	*charset = 1;
    if (!shift) {
	words[0] = entry & 0x1fu;			/* :302 */
	return 1;
    }
    words[0] = shift;
    words[1] = entry & 0x1fu;
    return 2;
}

/* the whole encoder call for one input byte: encoder kind FSK_B200_ENCODE_*; returns the words
 * stored (at most 2) */
FSK_HD unsigned int fsk_enc_byte(int kind, uint32_t *charset, unsigned int byte, uint32_t *words)
{
    if (kind != FSK_B200_ENCODE_BAUDOT) {
	words[0] = fsk_enc_ascii8(byte);
	return 1;
    }
    const int c = fsk_enc_toupper((int)(int8_t)(uint8_t)byte);
    return fsk_enc_baudot_with(charset, c, c >= 0 && c < 0x60 ? fsk_enc_baudot_entry(c) : 0u, words);
}

#endif
