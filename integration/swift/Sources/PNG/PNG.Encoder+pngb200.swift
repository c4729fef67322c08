//  PNG.Image.compress(stream:level:hint:) online on the device (Sources/PNG/PNG.Image.swift:576-668, PNG.Encoder.pull,
//  Sources/PNG/Encoding/PNG.Encoder.swift:33-129): the rows of the storage go in as bands, and the file comes out in
//  pieces -- head, IDAT chunks, IEND -- as soon as the reference would have written them.  Same shape as
//  PNG.DeviceContext: init, push, pop.
//  Written against the C ABI; NOT compiled in the pngb200 repository (its build image has no Swift toolchain).
import CPNGB200

extension PNG
{
    struct DeviceEncoder
    {
        private
        let handle:OpaquePointer
        private
        let stride:Int      // storage bytes a row

        /// The encoder of `image` at `level`; nothing is written until the first push.  `idatChunk` 0 gives the
        /// reference's 65 544-byte chunks (hint 1 << 15).
        init(image:PNG.Image, level:Int, idatChunk:Int = 0) throws
        {
            let (header, palette, _, transparency, cgbi):
                (PNG.Header, PNG.Palette?, PNG.Background?, PNG.Transparency?, [UInt8]?) = image.encode()
            var rgba:[UInt8] = []
            var desc:pngb200_png_encoder_desc = .init()
            desc.width              = UInt32.init(image.size.x)
            desc.height             = UInt32.init(image.size.y)
            desc.format.color       = header.pixel.code
            desc.format.depth       = UInt8.init(header.pixel.depth)
            desc.format.bgr         = cgbi == nil ? 0 : 1
            desc.interlaced         = image.layout.interlaced ? 1 : 0
            desc.level              = Int32.init(level)
            desc.idat_chunk         = UInt32.init(clamping: idatChunk)
            switch transparency
            {
            case .v(key: let v)?:
                desc.format.has_key = 1
                desc.format.key.0   = v
            case .rgb(key: let c)?:
                desc.format.has_key = 1
                (desc.format.key.0, desc.format.key.1, desc.format.key.2) = cgbi == nil ? (c.r, c.g, c.b) : (c.b, c.g, c.r)
            case .palette(alpha: let alpha)?:
                rgba = palette.map { $0.entries.enumerated().flatMap
                    { [$0.element.r, $0.element.g, $0.element.b, $0.offset < alpha.count ? alpha[$0.offset] : 255] } } ?? []
            case nil:
                rgba = palette.map { $0.entries.flatMap { [$0.r, $0.g, $0.b, 255] } } ?? []
            }
            desc.format.palette_count = UInt16.init(rgba.count / 4)
            let handle:OpaquePointer? = rgba.withUnsafeBufferPointer
            {
                desc.format.palette = $0.baseAddress      // read during the call
                return pngb200_png_encoder_create(LZ77.GPU.shared.ctx, &desc)
            }
            guard let handle:OpaquePointer
            else
            {
                throw pngb200Error(status: PNGB200_ERR_BAD_ARGUMENT.rawValue, 0, 0)
            }
            self.handle = handle
            self.stride = image.storage.count / max(1, image.size.y)
        }

        /// The next storage rows `rows` of `image`, top to bottom
        mutating
        func push(rows:Range<Int>, of image:PNG.Image) throws
        {
            let status:Int32 = image.storage.withUnsafeBufferPointer
            {
                pngb200_png_encoder_push(self.handle, $0.baseAddress.map { $0 + rows.lowerBound * self.stride },
                    rows.count * self.stride, Int32.init(PNGB200_MEM_HOST.rawValue))
            }
            guard status == 0
            else
            {
                throw pngb200Error(status: status, 0, 0)
            }
        }

        /// The next piece of the file, or nil when there is none yet
        mutating
        func pop() -> [UInt8]?
        {
            var bytes:UnsafePointer<UInt8>? = nil
            var count:Int = 0
            guard pngb200_png_encoder_pop(self.handle, &bytes, &count) == 1
            else
            {
                return nil
            }
            return .init(UnsafeBufferPointer<UInt8>.init(start: bytes, count: count))
        }

        func destroy()
        {
            pngb200_png_encoder_destroy(self.handle)
        }

        private
        init(handle:OpaquePointer, stride:Int)
        {
            self.handle = handle
            self.stride = stride
        }
        /// An independent copy (pngb200_png_encoder_clone) with its own copy of the pieces not popped yet.  The copy has
        /// a lifetime of its own: destroy both.
        func copy() -> Self?
        {
            guard let handle:OpaquePointer = pngb200_png_encoder_clone(self.handle)
            else
            {
                return nil
            }
            return .init(handle: handle, stride: self.stride)
        }
    }
}

extension PNG.Image
{
    /// compress(stream:level:hint:) with the row loop, deflate and IDAT framing on the device.  `hint` sets the IDAT
    /// chunk size as in Deflator+pngb200.swift (2 * hint bytes; 65 544 for the default 1 << 15).  The metadata chunks
    /// of `self.metadata` (cHRM, gAMA, sRGB, iCCP, sBIT, bKGD, hIST, pHYs, tIME, iTXt, sPLT, application chunks) are
    /// DROPPED by this body: a caller that needs them writes them behind the first piece (the head), as
    /// INTEGRATION §4c says.
    func compress<Destination>(stream:inout Destination, level:Int = 9, hint:Int = 1 << 15) throws
        where Destination:PNG.BytestreamDestination
    {
        let hint:Int = max(1, min(hint, 0x7f_ff_ff_ff))     // as PNG.Encoder.init clamps it
        var encoder:PNG.DeviceEncoder = try .init(image: self, level: level, idatChunk: hint == 1 << 15 ? 0 : 2 * hint)
        defer
        {
            encoder.destroy()
        }
        let band:Int = max(1, (1 << 20) / max(1, self.storage.count / max(1, self.size.y)))
        for y:Int in Swift.stride(from: 0, to: self.size.y, by: band)
        {
            try encoder.push(rows: y ..< min(self.size.y, y + band), of: self)
            while let piece:[UInt8] = encoder.pop()
            {
                try stream.write(piece)
            }
        }
    }
}
