//  PNG.Context on the device (Sources/PNG/Decoding/PNG.Context.swift): online decoding with the pixels assigned, and
//  overdrawn, by the GPU as each IDAT chunk arrives.  Same API shape as PNG.Context: init, push(data:overdraw:),
//  push(ancillary:) with IEND, and the image storage, which is a valid partial image after every push.
import CPNGB200

extension PNG
{
    struct DeviceContext
    {
        private
        let handle:OpaquePointer
        /// PNG.Image.storage, zero-filled at init (PNG.Context.init(..., uninitialized: false))
        private(set)
        var storage:UnsafeMutableBufferPointer<UInt8>

        init?(standard:PNG.Standard, header:PNG.Header, layout:PNG.Layout)
        {
            let count:Int = header.size.x * header.size.y * ((layout.format.pixel.volume + 7) >> 3)
            self.storage = .allocate(capacity: count)
            var desc:pngb200_png_context_desc = .init()
            desc.pixels     = UnsafeMutableRawPointer.init(self.storage.baseAddress)
            desc.pixels_cap = count
            desc.width      = UInt32.init(header.size.x)
            desc.height     = UInt32.init(header.size.y)
            desc.volume     = UInt8.init(layout.format.pixel.volume)
            desc.depth      = UInt8.init(layout.format.pixel.depth)
            desc.interlaced = layout.interlaced ? 1 : 0
            desc.standard   = standard == .ios ? 1 : 0
            desc.memspace   = Int32.init(PNGB200_MEM_HOST.rawValue)
            guard let handle:OpaquePointer = pngb200_png_context_create(LZ77.GPU.shared.ctx, &desc)
            else
            {
                self.storage.deallocate()
                return nil
            }
            self.handle = handle
        }

        /// PNG.Context.push(data:overdraw:) (PNG.Context.swift:76-100); the storage holds the new rows on return
        mutating
        func push(data:[UInt8], overdraw:Bool = false) throws
        {
            let status:Int32 = data.withUnsafeBufferPointer
            {
                pngb200_png_context_push(self.handle, $0.baseAddress, $0.count, overdraw ? 1 : 0)
            }
            if let error:any Error = self.error(status: status)
            {
                throw error
            }
        }

        /// Many pushes in one call (pngb200_png_context_push_batch), one per context, each context at most once: for a
        /// caller with many images in flight.  Returns, per push, the error push(data:overdraw:) would throw for it, or
        /// nil; throws only when the call itself fails.
        static
        func push(_ pushes:[(context:DeviceContext, data:[UInt8], overdraw:Bool)]) throws -> [(any Error)?]
        {
            let bytes:[UInt8] = pushes.flatMap(\.data)
            var descs:[pngb200_png_push_desc] = []
            let status:Int32 = bytes.withUnsafeBufferPointer
            {
                (bytes:UnsafeBufferPointer<UInt8>) in
                var offset:Int = 0
                for push:(context:DeviceContext, data:[UInt8], overdraw:Bool) in pushes
                {
                    var desc:pngb200_png_push_desc = .init()
                    desc.context  = push.context.handle
                    desc.data     = bytes.baseAddress.map { $0 + offset }
                    desc.n        = push.data.count
                    desc.overdraw = push.overdraw ? 1 : 0
                    descs.append(desc)
                    offset       += push.data.count
                }
                return pngb200_png_context_push_batch(LZ77.GPU.shared.ctx, &descs, descs.count)
            }
            guard status == 0
            else
            {
                throw pngb200Error(status: status, 0, 0)
            }
            return zip(pushes, descs).map { $0.context.error(status: $1.status) }
        }

        /// the error push(data:overdraw:) throws for a push status, or nil
        private
        func error(status:Int32) -> (any Error)?
        {
            switch status
            {
            case 0:     return nil
            case -48:   return PNG.DecodingError.extraneousImageData                      // PNG.Decoder.swift:142-147
            case -49:   return PNG.DecodingError.extraneousImageDataCompressedData         // :51-55
            default:
                var s:Int32 = 0, a:UInt32 = 0, b:UInt32 = 0
                pngb200_png_context_error(self.handle, &s, &a, &b)
                return pngb200Error(status: status, a, b)                                 // LZ77 errors, as the inflator
            }
        }

        /// push(ancillary:) with IEND (PNG.Context.swift:134-141)
        func end() throws
        {
            guard pngb200_png_context_end(self.handle) == 0
            else
            {
                throw PNG.DecodingError.incompleteImageDataCompressedDatastream
            }
        }

        /// the storage rows the last push wrote: what a viewer redraws
        var band:Range<Int>
        {
            var out:(UInt64, UInt64, UInt64, UInt64, UInt64, UInt64) = (0, 0, 0, 0, 0, 0)
            withUnsafeMutableBytes(of: &out)
            {
                _ = pngb200_png_context_progress(self.handle, $0.baseAddress!.assumingMemoryBound(to: UInt64.self))
            }
            return Int.init(out.4) ..< Int.init(out.5)
        }

        func destroy()
        {
            pngb200_png_context_destroy(self.handle)
            self.storage.deallocate()
        }

        private
        init(handle:OpaquePointer, storage:UnsafeMutableBufferPointer<UInt8>)
        {
            self.handle = handle
            self.storage = storage
        }
        /// An independent copy (pngb200_png_context_clone), its storage starting as this one's.  `storage`, of at least
        /// this context's storage bytes, becomes the copy's and is deallocated by its `destroy()`; nil allocates it.
        /// On failure (nil) a caller's `storage` stays the caller's.  The copy has a lifetime of its own: destroy both.
        func copy(storage given:UnsafeMutableBufferPointer<UInt8>? = nil) -> Self?
        {
            let storage:UnsafeMutableBufferPointer<UInt8> = given ?? .allocate(capacity: self.storage.count)
            guard let handle:OpaquePointer = pngb200_png_context_clone(self.handle,
                UnsafeMutableRawPointer.init(storage.baseAddress), storage.count)
            else
            {
                if  given == nil
                {
                    storage.deallocate()
                }
                return nil
            }
            return .init(handle: handle, storage: storage)
        }
    }
}
